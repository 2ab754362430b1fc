"""Autoregressive generation with a KV cache for the decoder-only models of this package (`LlamaForCausalLM`, `MixtralForCausalLM`,
`GPTForCausalLM`).

Role parity: the serving path the reference builds out of `masked_multihead_attention` / `block_multihead_attention` +
`FusedMultiTransformer` (python/paddle/incubate/nn/layer/fused_transformer.py) and PaddleNLP's `generate()`: prefill once, then one
token per step against cached keys / values, greedy or sampled (temperature, top-k, top-p), ragged prompts, early stop on EOS.

The cache layout is the decode kernel's: `k`, `v` of every layer are [B, H_kv, S_max, D] with `lens[b]` valid positions
(csrc/decode_attention.cu).  Prefill runs the model's own sublayers (fused RMSNorm / packed rotary / flash attention on CUDA) and writes
the rotated keys and the values into the cache; a decode step projects ONE token, rotates it at position `lens[b]`, appends it and attends
to the cache - through `decode_attention` (split-K over the cached positions) when `FLAGS_b200_decode_kernel` is set and the shapes qualify
(CUDA, head_dim 128 or 64, fp16 / bf16), otherwise through a masked softmax over the cache (any device / dtype; the default until the kernel
path has been exercised end to end on hardware)."""
from __future__ import annotations

import math

import torch

from ..tensor import Tensor


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


def _w(t):
    return t.as_subclass(Tensor) if isinstance(t, torch.Tensor) and not isinstance(t, Tensor) else t


class KVCache:
    """Per-layer key / value cache [B, H_kv, S_max, D] + the number of valid positions per sequence."""

    def __init__(self, num_layers, batch, kv_heads, max_len, head_dim, dtype, device):
        self.k = [torch.zeros(batch, kv_heads, max_len, head_dim, dtype=dtype, device=device) for _ in range(num_layers)]
        self.v = [torch.zeros(batch, kv_heads, max_len, head_dim, dtype=dtype, device=device) for _ in range(num_layers)]
        self.lens = torch.zeros(batch, dtype=torch.int32, device=device)
        self.max_len = max_len

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in self.k + self.v)

    def write_prefix(self, layer, k, v):
        """k, v: [B, S, H_kv, D] of the prompt (positions 0 .. S-1)."""
        s = k.shape[1]
        self.k[layer][:, :, :s] = k.transpose(1, 2)
        self.v[layer][:, :, :s] = v.transpose(1, 2)

    def append(self, layer, k, v):
        """k, v: [B, H_kv, D] of the new token; lands at position lens[b] of every sequence."""
        idx = self.lens.long()
        b = torch.arange(k.shape[0], device=k.device)
        self.k[layer][b, :, idx] = k
        self.v[layer][b, :, idx] = v


def _attend_cache(q, kc, vc, lens, scale, window=None):
    """q [B, H, D] against the cache [B, H_kv, S_max, D] with `lens` valid positions (the new token already appended); `window`: only the
    last `window` of them (sliding-window attention)."""
    from ..framework.flags import flag

    if flag("FLAGS_b200_decode_kernel", False) and q.is_cuda and q.shape[-1] in (64, 128) and q.dtype in (torch.float16, torch.bfloat16):
        from .._build import ext

        return ext().decode_attention(q.contiguous(), kc, vc, lens.to(torch.int32).contiguous(), float(scale), window or 0)
    b, h, d = q.shape
    hkv = kc.shape[1]
    smax = int(lens.max().item())
    k = kc[:, :, :smax].float()
    v = vc[:, :, :smax].float()
    if hkv != h:
        k = k.repeat_interleave(h // hkv, 1)
        v = v.repeat_interleave(h // hkv, 1)
    s = torch.einsum("bhd,bhsd->bhs", q.float(), k) * scale
    pos = torch.arange(smax, device=q.device)[None, None, :]
    mask = pos >= lens.long()[:, None, None]
    if window is not None:
        mask = mask | (pos < lens.long()[:, None, None] - window)
    s = s.masked_fill(mask, float("-inf"))
    return torch.einsum("bhs,bhsd->bhd", torch.softmax(s, -1), v).to(q.dtype)


class DecoderAdapter:
    """What generation needs from a decoder-only model of this package: embedding, decoder layers (each with `input_layernorm`, `self_attn`
    = LlamaAttention, `post_attention_layernorm` and a feed-forward), the output head.  Llama (dense SwiGLU MLP) and Mixtral (MoE
    feed-forward: routing is per token, so cached decoding equals recomputation) are supported."""

    def __init__(self, model):
        from . import llama as L

        self.model, self.L = model, L
        if hasattr(model, "llama"):
            self.cfg = model.config
            self.layers = list(model.llama.layers)
            self.embed = model.llama.embedding
            self.head = model.lm_head
            self.ffn = lambda layer, x: layer.mlp.down_proj(L.KA.swiglu(layer.mlp.gate_up_proj(x)))
        elif hasattr(model, "embed_tokens") and hasattr(model, "layers") and hasattr(list(model.layers)[0], "moe"):
            self.cfg = model.cfg
            self.layers = list(model.layers)
            self.embed = model.embed_tokens
            self.head = lambda h: model.lm_head(model.norm(h))
            self.ffn = lambda layer, x: layer.moe(x)
        else:
            raise NotImplementedError(f"generation does not know the layout of {type(model).__name__}")
        at = self.layers[0].self_attn
        if at.mp != 1:
            raise NotImplementedError("generation serves a single-rank replica (mp_degree 1)")
        self.nh, self.nkv, self.hd = at.num_heads, at.num_kv_heads, at.head_dim

    # -- the three pieces a packed-batch engine (models/serving.py) needs; tokens are [1, T], positions [1, T]
    def embed_tokens(self, ids, position_ids):
        return self.embed(_w(ids))

    def attn_in(self, layer, h, position_ids):
        """-> packed q | k | v of every token [1, T, (H + 2 H_kv) * D] (normed, projected, rotated)."""
        L = self.L
        if not hasattr(self, "_rope"):
            self._rope = L.rope_cache(self.cfg, _raw(h).device)
        cos, sin = self._rope
        nh, nkv, hd = self.nh, self.nkv, self.hd
        return _raw(L.KR.apply_rope_packed(layer.self_attn.qkv_proj(layer.input_layernorm(h)), cos, sin, nh + nkv, nh + 2 * nkv, hd, position_ids, neox=True))

    def attn_out(self, layer, h, a):
        """Attention output [1, T, H * D] -> the layer's output."""
        a = layer.self_attn.o_proj(_w(a))
        x, h = layer.post_attention_layernorm(a, residual=h)
        return h + self.ffn(layer, x)

    def logits(self, h):
        return _raw(self.head(_w(h)))


class GPTAdapter:
    """The same interface for `GPTForCausalLM` (learned positions, LayerNorm, biased packed qkv, GELU MLP, tied head)."""

    def __init__(self, model):
        self.model, self.cfg = model, model.cfg
        self.layers = list(model.gpt.blocks)
        self.nh = self.nkv = self.cfg.num_attention_heads
        self.hd = self.cfg.head_dim

    def embed_tokens(self, ids, position_ids):
        g = self.model.gpt
        if int(position_ids.max()) >= self.cfg.max_position_embeddings:
            raise ValueError(f"position {int(position_ids.max())} is outside the model's {self.cfg.max_position_embeddings} learned positions")
        return g.wte(_w(ids)) + g.wpe(_w(position_ids))

    def attn_in(self, blk, h, position_ids):
        return _raw(blk.qkv(blk.ln1(h)))                   # [.., 3, H, D] flattened: q | k | v per token

    def attn_out(self, blk, h, a):
        from ..nn import functional as F

        h = h + blk.proj(_w(a))
        return h + blk.fc2(F.gelu(blk.fc1(blk.ln2(h))))

    def logits(self, h):
        g = self.model.gpt
        return _raw(g.wte(g.ln_f(_w(h)), project=True))


def make_adapter(model):
    if hasattr(model, "gpt") and hasattr(model.gpt, "blocks"):
        return GPTAdapter(model)
    return DecoderAdapter(model)


class LlamaGenerator:
    """Prefill + decode over the sublayers of a decoder-only model (`LlamaForCausalLM`, `MixtralForCausalLM`); no tensor / pipeline
    parallelism: serve one replica per GPU."""

    def __init__(self, model):
        ad = DecoderAdapter(model)
        self.ad, self.model, self.cfg, self.layers = ad, model, ad.cfg, ad.layers
        self.nh, self.nkv, self.hd = ad.nh, ad.nkv, ad.hd
        self._rope = ad.L.rope_cache
        self._KR = ad.L.KR
        self.window = getattr(self.cfg, "sliding_window", None)

    # -- one decoder layer on [B, S, hidden] with explicit positions; returns (h, k, v) with k, v [B, S, H_kv, D] (k rotated)
    def _layer(self, layer, h, cos, sin, position_ids, attend):
        at = layer.self_attn
        nh, nkv, hd = self.nh, self.nkv, self.hd
        x = layer.input_layernorm(h)
        qkv = _raw(self._KR.apply_rope_packed(at.qkv_proj(x), cos, sin, nh + nkv, nh + 2 * nkv, hd, position_ids, neox=True))
        b, s = qkv.shape[0], qkv.shape[1]
        qkv = qkv.reshape(b, s, nh + 2 * nkv, hd)
        q, k, v = qkv[:, :, :nh], qkv[:, :, nh:nh + nkv], qkv[:, :, nh + nkv:]
        a = attend(q, k, v)                                               # [B, S, H, D]
        a = at.o_proj(_w(a.reshape(b, s, nh * hd)))
        x, h = layer.post_attention_layernorm(a, residual=h)
        return h + self.ad.ffn(layer, x), k, v

    @torch.no_grad()
    def prefill(self, input_ids, prompt_lens, cache):
        """Whole prompts (right padded to a common length) through the stack; fills the cache; returns the logits of every sequence's
        LAST real token [B, vocab]."""
        ids = _raw(input_ids)
        b, s = ids.shape
        scale = 1.0 / math.sqrt(self.hd)
        h = self.ad.embed(_w(ids))
        cos, sin = self._rope(self.cfg, _raw(h).device)
        pos = torch.arange(s, device=ids.device, dtype=torch.int64).unsqueeze(0).expand(b, s).contiguous()

        mask = None if self.window is None else self.ad.L.window_mask(s, s, self.window, ids.device)

        def attend(q, k, v):
            rep = self.nh // self.nkv
            kk, vv = (k.repeat_interleave(rep, 2), v.repeat_interleave(rep, 2)) if rep > 1 else (k, v)
            o = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), kk.transpose(1, 2), vv.transpose(1, 2), attn_mask=mask,
                                                                 is_causal=mask is None, scale=scale)
            return o.transpose(1, 2)

        for i, layer in enumerate(self.layers):
            h, k, v = self._layer(layer, h, cos, sin, pos, attend)
            cache.write_prefix(i, k, v)
        cache.lens.copy_(prompt_lens.to(torch.int32))
        last = (prompt_lens.long() - 1).clamp(min=0)
        hl = _raw(h)[torch.arange(b, device=ids.device), last].unsqueeze(1)   # [B, 1, hidden]
        return _raw(self.ad.head(_w(hl)))[:, 0]

    @torch.no_grad()
    def decode_step(self, tokens, cache):
        """One new token per sequence ([B] ids) at position cache.lens[b]; returns logits [B, vocab] and advances the cache."""
        ids = _raw(tokens).reshape(-1, 1)
        b = ids.shape[0]
        scale = 1.0 / math.sqrt(self.hd)
        h = self.ad.embed(_w(ids))
        cos, sin = self._rope(self.cfg, _raw(h).device)
        pos = cache.lens.long().reshape(b, 1)
        for i, layer in enumerate(self.layers):
            def attend(q, k, v, i=i):
                cache.append(i, k[:, 0], v[:, 0])
                return _attend_cache(q[:, 0], cache.k[i], cache.v[i], cache.lens + 1, scale, self.window).unsqueeze(1)

            h, _, _ = self._layer(layer, h, cos, sin, pos, attend)
        cache.lens += 1
        return _raw(self.ad.head(h))[:, 0]


class GPTGenerator:
    """Prefill + decode for `GPTForCausalLM` (models/gpt.py): learned absolute positions, LayerNorm, packed [3, H, D] qkv projection with
    bias, GELU MLP, LM head tied to the token embedding.  Same interface as LlamaGenerator."""

    def __init__(self, model):
        self.model, self.cfg = model, model.cfg
        self.layers = list(model.gpt.blocks)
        self.nh = self.nkv = self.cfg.num_attention_heads
        self.hd = self.cfg.head_dim

    def _layer(self, blk, h, attend):
        from ..nn import functional as F

        b, s, hid = h.shape
        qkv = _raw(blk.qkv(blk.ln1(h))).reshape(b, s, 3, self.nh, self.hd)
        a = attend(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2])
        h = h + blk.proj(_w(a.reshape(b, s, hid)))
        return h + blk.fc2(F.gelu(blk.fc1(blk.ln2(h)))), qkv[:, :, 1], qkv[:, :, 2]

    def _embed(self, ids, pos):
        g = self.model.gpt
        if int(pos.max()) >= self.cfg.max_position_embeddings:
            raise ValueError(f"position {int(pos.max())} is outside the model's {self.cfg.max_position_embeddings} learned positions")
        return g.wte(_w(ids)) + g.wpe(_w(pos))

    def _head(self, h):
        g = self.model.gpt
        return _raw(g.wte(g.ln_f(h), project=True))

    @torch.no_grad()
    def prefill(self, input_ids, prompt_lens, cache):
        ids = _raw(input_ids)
        b, s = ids.shape
        scale = 1.0 / math.sqrt(self.hd)
        h = self._embed(ids, torch.arange(s, device=ids.device, dtype=torch.int64).unsqueeze(0).expand(b, s))

        def attend(q, k, v):
            o = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=True, scale=scale)
            return o.transpose(1, 2)

        for i, blk in enumerate(self.layers):
            h, k, v = self._layer(blk, h, attend)
            cache.write_prefix(i, k, v)
        cache.lens.copy_(prompt_lens.to(torch.int32))
        last = (prompt_lens.long() - 1).clamp(min=0)
        hl = _raw(h)[torch.arange(b, device=ids.device), last].unsqueeze(1)
        return self._head(_w(hl))[:, 0]

    @torch.no_grad()
    def decode_step(self, tokens, cache):
        ids = _raw(tokens).reshape(-1, 1)
        b = ids.shape[0]
        scale = 1.0 / math.sqrt(self.hd)
        h = self._embed(ids, cache.lens.long().reshape(b, 1))
        for i, blk in enumerate(self.layers):
            def attend(q, k, v, i=i):
                cache.append(i, k[:, 0], v[:, 0])
                return _attend_cache(q[:, 0], cache.k[i], cache.v[i], cache.lens + 1, scale).unsqueeze(1)

            h, _, _ = self._layer(blk, h, attend)
        cache.lens += 1
        return self._head(h)[:, 0]


def make_generator(model):
    """The generator for a decoder-only model of this package."""
    if hasattr(model, "gpt") and hasattr(model.gpt, "blocks"):
        return GPTGenerator(model)
    return LlamaGenerator(model)


def _sample(logits, do_sample, temperature, top_k, top_p, generator=None):
    if not do_sample or temperature == 0.0:
        return logits.argmax(-1)
    logits = logits.float() / max(float(temperature), 1e-6)
    if top_k and top_k > 0:
        kth = torch.topk(logits, min(int(top_k), logits.shape[-1]), dim=-1).values[..., -1:]
        logits = logits.masked_fill(logits < kth, float("-inf"))
    if top_p is not None and top_p < 1.0:
        sorted_logits, order = torch.sort(logits, descending=True, dim=-1)
        probs = torch.softmax(sorted_logits, -1)
        drop = probs.cumsum(-1) - probs > top_p                       # keep the smallest prefix whose mass reaches top_p
        sorted_logits = sorted_logits.masked_fill(drop, float("-inf"))
        logits = torch.full_like(logits, float("-inf")).scatter(-1, order, sorted_logits)
    return torch.multinomial(torch.softmax(logits, -1), 1, generator=generator).squeeze(-1)


@torch.no_grad()
def generate(model, input_ids, max_new_tokens=32, prompt_lens=None, do_sample=False, temperature=1.0, top_k=0, top_p=1.0, eos_token_id=None, pad_token_id=0,
             max_length=None, return_cache=False):
    """Generate up to `max_new_tokens` tokens per sequence.  `input_ids` [B, S] (right padded when `prompt_lens` [B] is given).
    Returns ids [B, S_max_prompt + new] where position `prompt_lens[b] + t` holds the t-th generated token of sequence b (the padding
    of shorter prompts is overwritten), padded with `pad_token_id` after an EOS."""
    was_training = model.training
    model.eval()
    try:
        ids = _raw(input_ids).long()
        b, s = ids.shape
        dev = ids.device
        lens = torch.full((b,), s, dtype=torch.int64, device=dev) if prompt_lens is None else _raw(prompt_lens).to(dev).long()
        total = int(max_length) if max_length is not None else s + int(max_new_tokens)
        gen = make_generator(model)
        p0 = next(iter(model.parameters()))
        cache = KVCache(len(gen.layers), b, gen.nkv, total, gen.hd, _raw(p0).dtype, dev)
        out = torch.full((b, total), int(pad_token_id), dtype=torch.int64, device=dev)
        for i in range(b):
            out[i, : int(lens[i])] = ids[i, : int(lens[i])]
        logits = gen.prefill(ids, lens, cache)
        done = torch.zeros(b, dtype=torch.bool, device=dev)
        rows = torch.arange(b, device=dev)
        steps = min(int(max_new_tokens), total - int(lens.min()))
        for t in range(steps):
            nxt = _sample(logits, do_sample, temperature, top_k, top_p)
            nxt = torch.where(done, torch.full_like(nxt, int(pad_token_id)), nxt)
            pos = (lens + t).clamp(max=total - 1)
            out[rows, pos] = torch.where(lens + t < total, nxt, out[rows, pos])
            if eos_token_id is not None:
                done = done | (nxt == int(eos_token_id))
                if bool(done.all()):
                    break
            if t + 1 < steps and int(cache.lens.max()) < total:
                logits = gen.decode_step(nxt, cache)
        res = _w(out)
        return (res, cache) if return_cache else res
    finally:
        if was_training:
            model.train()
