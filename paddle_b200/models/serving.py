"""Continuous-batching generation engine over a paged KV cache.

Role parity: the serving stack the reference assembles from `block_multihead_attention` (paged KV cache + block tables,
paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu) and its in-flight batching scheduler: requests join and leave the
running batch between steps, the KV cache is a pool of fixed-size blocks handed out on demand, and a sequence that cannot get a block is
preempted (its blocks go back to the pool; it is re-prefilled later from prompt + generated tokens).

Every step packs the tokens of all scheduled sequences into ONE [tokens, hidden] batch: whole prompts for the sequences being prefilled,
one token for the sequences being decoded.  The decoder layers run on the packed batch with the model's own sublayers; attention is
`incubate.nn.paged_attention.block_attention` - on CUDA (head_dim 128, fp16 / bf16) one indexed scatter of the new K / V rows into the
block pool, `decode_attention_paged` for the decode rows and one paged wgmma prefill attention (`attention_fwd_paged`) for the prefill rows.

Chunked prefill (`max_prefill_chunk=N`): an admitted prompt still gets the blocks for its whole length, but is fed over successive steps,
at most N tokens (and no more than the step's remaining token budget) at a time, each chunk attending to the chunks already cached.  Decode
rows are scheduled first, so long prompts no longer stall running sequences, and a prompt longer than `max_batch_tokens` can be served.
A sequence samples its first token after its last chunk.

Quantized KV cache (`kv_cache_dtype="int8"` or `"float8_e4m3fn"`): the block pool stores one byte per element, so the same memory holds
twice the tokens of a 16-bit cache and decode reads half the bytes.  The scales are static, one per KV head and layer, derived from a
calibrated absmax `kv_cache_absmax` [num_layers, 2, H_kv] (see `calibrate_kv_cache`): quant_scale = 1 / absmax and dequant_scale =
absmax / bound, with bound 127 (int8) or 448 (fp8).  Static scales make chunked prefill and preemption work unchanged.
"""
from __future__ import annotations

import torch

from ..incubate.nn.paged_attention import block_attention
from .generation import _raw, _sample, _w


class BlockAllocator:
    """Pool of KV-cache blocks (ids 0 .. num_blocks-1)."""

    def __init__(self, num_blocks):
        self.num_blocks = int(num_blocks)
        self._free = list(range(self.num_blocks - 1, -1, -1))

    def num_free(self):
        return len(self._free)

    def alloc(self):
        if not self._free:
            raise MemoryError("KV-cache block pool is exhausted")
        return self._free.pop()

    def free(self, blocks):
        self._free.extend(reversed(blocks))


class Sequence:
    WAITING, RUNNING, FINISHED = "waiting", "running", "finished"

    def __init__(self, seq_id, prompt, max_new_tokens, eos_token_id=None, do_sample=False, temperature=1.0, top_k=0, top_p=1.0):
        self.id, self.prompt, self.max_new_tokens, self.eos = seq_id, [int(t) for t in prompt], int(max_new_tokens), eos_token_id
        self.do_sample, self.temperature, self.top_k, self.top_p = do_sample, temperature, top_k, top_p
        self.generated, self.blocks, self.cached, self.status, self.preemptions = [], [], 0, Sequence.WAITING, 0
        self.target = 0                            # tokens to prefill since admission: the sequence samples once cached reaches it

    def tokens(self):
        return self.prompt + self.generated

    def finished(self):
        return self.status == Sequence.FINISHED


_KV_CACHE_DTYPES = {"int8": (torch.int8, 127.0), "float8_e4m3fn": (torch.float8_e4m3fn, 448.0)}


class LLMEngine:
    """add_request() any time; step() runs one scheduler iteration (admit / preempt, one packed forward, one token per running sequence)."""

    def __init__(self, model, num_blocks=256, block_size=16, max_running=64, max_batch_tokens=8192, max_prefill_chunk=None, kv_cache_dtype=None,
                 kv_cache_absmax=None):
        from .generation import make_adapter

        model.eval()
        ad = make_adapter(model)                   # Llama (dense), Mixtral (MoE) and GPT layouts
        self.ad, self.model, self.cfg, self.layers = ad, model, ad.cfg, ad.layers
        self.nh, self.nkv, self.hd = ad.nh, ad.nkv, ad.hd
        self.block_size, self.max_running, self.max_batch_tokens = int(block_size), int(max_running), int(max_batch_tokens)
        if max_prefill_chunk is not None and int(max_prefill_chunk) < 1:
            raise ValueError(f"max_prefill_chunk must be a positive number of tokens or None, got {max_prefill_chunk}")
        self.max_prefill_chunk = None if max_prefill_chunk is None else int(max_prefill_chunk)
        p0 = _raw(next(iter(model.parameters())))
        self.device, self.dtype = p0.device, p0.dtype
        self.alloc = BlockAllocator(num_blocks)
        self._kv_quant = [{} for _ in self.layers]       # per layer: block_attention's cache quantization arguments
        cache_dtype = self.dtype
        if kv_cache_dtype is not None:
            cache_dtype, self._kv_quant = self._static_kv_quant(kv_cache_dtype, kv_cache_absmax)
        elif kv_cache_absmax is not None:
            raise ValueError("kv_cache_absmax is only used with kv_cache_dtype='int8' or 'float8_e4m3fn'")
        self.kv_cache_dtype = cache_dtype
        shape = (num_blocks, self.nkv, self.block_size, self.hd)
        self.key_cache = [torch.zeros(shape, dtype=cache_dtype, device=self.device) for _ in self.layers]
        self.value_cache = [torch.zeros(shape, dtype=cache_dtype, device=self.device) for _ in self.layers]
        self._observe = None                             # calibrate_kv_cache: called with (layer index, packed qkv rows) every forward
        self.waiting, self.running, self.done = [], [], {}
        self._next_id = 0
        self.stats = {"steps": 0, "prefill_tokens": 0, "decode_tokens": 0, "preemptions": 0, "max_running": 0}

    def _static_kv_quant(self, kv_cache_dtype, absmax):
        name = str(kv_cache_dtype).replace("torch.", "")
        if name not in _KV_CACHE_DTYPES:
            raise ValueError(f"kv_cache_dtype must be None, 'int8' or 'float8_e4m3fn', got {kv_cache_dtype!r}")
        dtype, bound = _KV_CACHE_DTYPES[name]
        shape = (len(self.layers), 2, self.nkv)
        if absmax is None or tuple(_raw(absmax).shape) != shape:
            raise ValueError(f"kv_cache_dtype={name!r} needs kv_cache_absmax of shape [num_layers, 2, H_kv] = {list(shape)} "
                             "(models.calibrate_kv_cache computes it)")
        am = _raw(absmax).to(self.device, torch.float32)
        am = torch.where(am > 0, am, torch.ones_like(am))   # a head whose rows are all zero: any scale stores them exactly
        qs, dq = 1.0 / am, am / bound
        quant = [{"cache_k_quant_scales": qs[li, 0], "cache_v_quant_scales": qs[li, 1], "cache_k_dequant_scales": dq[li, 0],
                  "cache_v_dequant_scales": dq[li, 1], "quant_max_bound": bound, "quant_min_bound": -bound} for li in range(len(self.layers))]
        return dtype, quant

    # ---- requests ---------------------------------------------------------------------------------------------------------------
    def add_request(self, prompt_ids, max_new_tokens=32, eos_token_id=None, do_sample=False, temperature=1.0, top_k=0, top_p=1.0):
        prompt = _raw(prompt_ids).reshape(-1).tolist() if isinstance(prompt_ids, torch.Tensor) else list(prompt_ids)
        need = (len(prompt) + max_new_tokens + self.block_size - 1) // self.block_size
        if need > self.alloc.num_blocks:
            raise ValueError(f"request needs {need} KV blocks, the pool has {self.alloc.num_blocks}")
        s = Sequence(self._next_id, prompt, max_new_tokens, eos_token_id, do_sample, temperature, top_k, top_p)
        self._next_id += 1
        self.waiting.append(s)
        return s.id

    def has_unfinished(self):
        return bool(self.waiting or self.running)

    # ---- scheduling -------------------------------------------------------------------------------------------------------------
    def _blocks_for(self, n_tokens):
        return (n_tokens + self.block_size - 1) // self.block_size

    def _preempt(self, s):
        self.alloc.free(s.blocks)
        s.blocks, s.cached, s.status = [], 0, Sequence.WAITING
        s.preemptions += 1
        self.stats["preemptions"] += 1
        self.running.remove(s)
        self.waiting.insert(0, s)              # first in line when blocks come back

    def _schedule(self):
        """Returns (decode sequences, [(prefill sequence, tokens this step)]).  Running sequences get their next slot first (newest ones are
        preempted when the pool runs dry); then half-prefilled sequences get their next chunk; then waiting sequences are admitted while
        blocks, the running limit and the token budget allow (whole prompts, or a first chunk with max_prefill_chunk)."""
        decode = []
        for s in list(self.running):
            if s not in self.running or s.cached < s.target:     # gone, or still prefilling (its blocks are already allocated)
                continue
            if self._blocks_for(s.cached + 1) > len(s.blocks):
                while self.alloc.num_free() == 0:
                    victim = next((v for v in reversed(self.running) if v is not s), None)
                    if victim is None:
                        break
                    self._preempt(victim)
                    if victim in decode:
                        decode.remove(victim)
                if self.alloc.num_free() == 0:
                    self._preempt(s)
                    continue
                s.blocks.append(self.alloc.alloc())
            decode.append(s)
        budget = self.max_batch_tokens - len(decode)
        chunk = self.max_prefill_chunk
        prefill = []
        for s in self.running:
            if s.cached < s.target and budget > 0:
                n = min(chunk, s.target - s.cached, budget)
                prefill.append((s, n))
                budget -= n
        admitted = 0
        while self.waiting and len(self.running) + admitted < self.max_running:
            s = self.waiting[0]
            total = len(s.tokens())
            n = total if chunk is None else min(chunk, total, budget)
            need = self._blocks_for(total + 1)
            if n > budget or (chunk is not None and budget == 0) or need > self.alloc.num_free():
                break
            self.waiting.pop(0)
            s.blocks = [self.alloc.alloc() for _ in range(need)]
            s.target = total
            prefill.append((s, n))
            admitted += 1
            budget -= n
        return decode, prefill

    # ---- one packed forward -------------------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _forward(self, seqs, n_new, enc, dec):
        dev = self.device
        toks, pos = [], []
        for s, n in zip(seqs, n_new):
            all_t = s.tokens()
            toks += all_t[s.cached:s.cached + n]
            pos += list(range(s.cached, s.cached + n))
        ids = torch.tensor(toks, dtype=torch.int64, device=dev).unsqueeze(0)                 # [1, T]
        position_ids = torch.tensor(pos, dtype=torch.int64, device=dev).unsqueeze(0)
        cu = torch.zeros(len(seqs) + 1, dtype=torch.int32, device=dev)
        cu[1:] = torch.cumsum(torch.tensor(n_new, dtype=torch.int32, device=dev), 0)
        max_blocks = max(len(s.blocks) for s in seqs)
        bt = torch.zeros(len(seqs), max_blocks, dtype=torch.int32, device=dev)
        for i, s in enumerate(seqs):
            bt[i, : len(s.blocks)] = torch.tensor(s.blocks, dtype=torch.int32, device=dev)
        enc_t = torch.tensor(enc, dtype=torch.int32, device=dev)
        dec_t = torch.tensor(dec, dtype=torch.int32, device=dev)
        now_t = torch.tensor(n_new, dtype=torch.int32, device=dev)
        nh, nkv, hd = self.nh, self.nkv, self.hd
        h = self.ad.embed_tokens(ids, position_ids)
        for li, layer in enumerate(self.layers):
            qkv = self.ad.attn_in(layer, h, position_ids)
            t = qkv.shape[1]
            if self._observe is not None:
                self._observe(li, qkv.reshape(t, (nh + 2 * nkv) * hd))
            out, _, _, _ = block_attention(qkv.reshape(t, (nh + 2 * nkv) * hd), self.key_cache[li], self.value_cache[li], enc_t, dec_t, now_t, cu, bt,
                                           self.block_size, **self._kv_quant[li])
            h = self.ad.attn_out(layer, h, _raw(out).reshape(1, t, nh * hd))
        last = (cu[1:].long() - 1)
        return self.ad.logits(_raw(h)[:, last])[0]                                     # [num_seqs, vocab]

    def step(self):
        """One iteration.  Returns [(request id, new token, finished)] for every sequence that produced a token."""
        decode, prefill = self._schedule()
        seqs = decode + [s for s, _ in prefill]
        if not seqs:
            if self.waiting and not self.running:
                raise MemoryError("the KV-cache pool cannot hold the next waiting request")
            return []
        n_new = [1] * len(decode) + [n for _, n in prefill]
        enc = [0] * len(decode) + [n if s.cached == 0 else 0 for s, n in prefill]     # a continuing chunk attends to its cached prefix
        dec = [s.cached for s in decode] + [s.cached for s, _ in prefill]
        logits = self._forward(seqs, n_new, enc, dec)
        self.stats["steps"] += 1
        self.stats["decode_tokens"] += len(decode)
        self.stats["prefill_tokens"] += sum(n_new[len(decode):])
        out = []
        for i, (s, n) in enumerate(zip(seqs, n_new)):
            s.cached += n
            if s.status != Sequence.RUNNING:
                s.status = Sequence.RUNNING
                self.running.append(s)
            if s.cached < s.target:                # more chunks to come: nothing to sample yet
                continue
            tok = int(_sample(logits[i: i + 1], s.do_sample, s.temperature, s.top_k, s.top_p)[0])
            s.generated.append(tok)
            fin = len(s.generated) >= s.max_new_tokens or (s.eos is not None and tok == s.eos)
            if fin:
                s.status = Sequence.FINISHED
                self.running.remove(s)
                self.alloc.free(s.blocks)
                s.blocks = []
                self.done[s.id] = s
            out.append((s.id, tok, fin))
        self.stats["max_running"] = max(self.stats["max_running"], len(self.running))
        return out

    def run_until_done(self, max_steps=100000):
        for _ in range(max_steps):
            if not self.has_unfinished():
                break
            self.step()
        return {i: s.generated for i, s in self.done.items()}

    def result(self, request_id):
        s = self.done.get(request_id)
        return None if s is None else _w(torch.tensor(s.generated, dtype=torch.int64))


@torch.no_grad()
def calibrate_kv_cache(model, prompts, block_size=16):
    """absmax [num_layers, 2, H_kv] (fp32) of exactly the rows LLMEngine writes into its KV cache when it prefills `prompts`: K after
    rotary, and V, per layer and KV head.  Pass it as LLMEngine(kv_cache_dtype=..., kv_cache_absmax=...)."""
    prompts = [_raw(p).reshape(-1).tolist() if isinstance(p, torch.Tensor) else list(p) for p in prompts]
    longest = max(len(p) for p in prompts)
    eng = LLMEngine(model, num_blocks=(longest + 1 + block_size - 1) // block_size, block_size=block_size, max_running=1,
                    max_batch_tokens=longest + 1)
    nh, nkv, hd = eng.nh, eng.nkv, eng.hd
    amax = torch.zeros(len(eng.layers), 2, nkv, dtype=torch.float32, device=eng.device)

    def observe(li, qkv):
        rows = qkv.reshape(qkv.shape[0], nh + 2 * nkv, hd).float()
        amax[li, 0] = torch.maximum(amax[li, 0], rows[:, nh:nh + nkv].abs().amax(dim=(0, 2)))
        amax[li, 1] = torch.maximum(amax[li, 1], rows[:, nh + nkv:].abs().amax(dim=(0, 2)))

    eng._observe = observe
    for p in prompts:
        eng.add_request(p, max_new_tokens=1)     # the first token is sampled from the prefill; its own row is never written
    eng.run_until_done()
    return amax
