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

Speculative decoding (`draft_model=..., num_speculative_tokens=k`): a greedy decode sequence gets k_s = min(k, tokens left - 1)
speculative slots, shrunk when the pool has too few free blocks for cached + k_s + 1 tokens (speculation never preempts) or the token
budget runs out (a row costs k_s + 1).  The draft - any model `make_adapter` supports, with its own caches over the target's block ids -
first catches up on every token its cache lacks (this step's prefill chunks of greedy sequences and 1-2 tokens per speculating row),
then runs k_s - 1 single-token forwards, proposing its argmax each time.  One target forward verifies every speculating row with
now = 1 + k_s tokens (block_attention sends those rows to `decode_attention_paged_multi`); the longest prefix of proposals equal to
the target's argmax is accepted, followed by the target's own token at the first mismatch (or the bonus token after a full match),
so greedy outputs equal non-speculative decoding.  Sampling requests decode one token per step as without a draft.
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
        self.draft_cached, self.spec = 0, 0        # speculative decoding: positions in the draft's cache, proposals this step

    def tokens(self):
        return self.prompt + self.generated

    def finished(self):
        return self.status == Sequence.FINISHED


_KV_CACHE_DTYPES = {"int8": (torch.int8, 127.0), "float8_e4m3fn": (torch.float8_e4m3fn, 448.0)}


class LLMEngine:
    """add_request() any time; step() runs one scheduler iteration (admit / preempt, one packed forward, one token per running sequence;
    with a draft model, up to num_speculative_tokens + 1 tokens per greedy decode sequence)."""

    def __init__(self, model, num_blocks=256, block_size=16, max_running=64, max_batch_tokens=8192, max_prefill_chunk=None, kv_cache_dtype=None,
                 kv_cache_absmax=None, draft_model=None, num_speculative_tokens=0):
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
        self._target = (ad, self.key_cache, self.value_cache, self._kv_quant)
        self.waiting, self.running, self.done = [], [], {}
        self._next_id = 0
        self.stats = {"steps": 0, "prefill_tokens": 0, "decode_tokens": 0, "preemptions": 0, "max_running": 0}
        self.num_speculative_tokens, self._draft = self._draft_setup(draft_model, num_speculative_tokens, num_blocks)
        if self.num_speculative_tokens:
            self.stats.update(draft_tokens=0, accepted_tokens=0)

    def _draft_setup(self, draft_model, k, num_blocks):
        """(k, (adapter, key caches, value caches, no quantization)) of the draft model, or (0, None) without one."""
        from .generation import make_adapter

        if draft_model is None:
            if k:
                raise ValueError(f"num_speculative_tokens={k} needs a draft_model")
            return 0, None
        if int(k) < 1:
            raise ValueError(f"a draft_model needs num_speculative_tokens >= 1, got {k}")
        draft_model.eval()
        dad = make_adapter(draft_model)
        if int(dad.cfg.vocab_size) != int(self.cfg.vocab_size):
            raise ValueError(f"the draft's vocab size {dad.cfg.vocab_size} differs from the target's {self.cfg.vocab_size}")
        dtype = _raw(next(iter(draft_model.parameters()))).dtype
        shape = (num_blocks, dad.nkv, self.block_size, dad.hd)          # the target's block ids name the same positions here
        kc = [torch.zeros(shape, dtype=dtype, device=self.device) for _ in dad.layers]
        vc = [torch.zeros(shape, dtype=dtype, device=self.device) for _ in dad.layers]
        return int(k), (dad, kc, vc, [{} for _ in dad.layers])

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
        s.blocks, s.cached, s.draft_cached, s.status = [], 0, 0, Sequence.WAITING
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
        if self.num_speculative_tokens:
            budget = self._assign_speculation(decode, budget)
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

    def _assign_speculation(self, decode, budget):
        """Sets each decode sequence's speculative slots k_s (0 for sampling requests), allocating blocks for cached + k_s + 1 tokens from
        free blocks only, and returns the token budget left."""
        for s in decode:
            k = 0 if s.do_sample else min(self.num_speculative_tokens, s.max_new_tokens - len(s.generated) - 1, budget)
            while k > 0 and self._blocks_for(s.cached + k + 1) - len(s.blocks) > self.alloc.num_free():
                k -= 1
            s.blocks += [self.alloc.alloc() for _ in range(self._blocks_for(s.cached + k + 1) - len(s.blocks))]
            s.spec = k
            budget -= k
        return budget

    # ---- one packed forward -------------------------------------------------------------------------------------------------------
    def _forward(self, seqs, n_new, enc, dec):
        """The target model over this step's rows (s.tokens() from s.cached); logits of each sequence's last row [num_seqs, vocab]."""
        return self._run(self._target, seqs, n_new, enc, dec)

    @torch.no_grad()
    def _run(self, net, seqs, n_new, enc, dec, toks=None, rows=None):
        """One packed forward of `net` = (adapter, key caches, value caches, quantization args) over the sequences' blocks: n_new[i] tokens
        at positions dec[i] ... (toks[i], by default taken from s.tokens()).  Returns the logits of packed rows `rows` (default: each
        sequence's last row)."""
        ad, key_cache, value_cache, kv_quant = net
        dev = self.device
        if toks is None:
            toks = [s.tokens()[p:p + n] for s, p, n in zip(seqs, dec, n_new)]
        pos = [i for p, n in zip(dec, n_new) for i in range(p, p + n)]
        toks = [t for tt in toks for t in tt]
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
        nh, nkv, hd = ad.nh, ad.nkv, ad.hd
        h = ad.embed_tokens(ids, position_ids)
        for li, layer in enumerate(ad.layers):
            qkv = ad.attn_in(layer, h, position_ids)
            t = qkv.shape[1]
            if self._observe is not None and net is self._target:
                self._observe(li, qkv.reshape(t, (nh + 2 * nkv) * hd))
            out, _, _, _ = block_attention(qkv.reshape(t, (nh + 2 * nkv) * hd), key_cache[li], value_cache[li], enc_t, dec_t, now_t, cu, bt,
                                           self.block_size, **kv_quant[li])
            h = ad.attn_out(layer, h, _raw(out).reshape(1, t, nh * hd))
        rows = (cu[1:].long() - 1) if rows is None else torch.tensor(rows, dtype=torch.int64, device=dev)
        return ad.logits(_raw(h)[:, rows])[0]                                          # [len(rows), vocab]

    def _finish_token(self, s, tok):
        """Appends a generated token; returns whether the sequence finished (its blocks go back to the pool)."""
        s.generated.append(tok)
        fin = len(s.generated) >= s.max_new_tokens or (s.eos is not None and tok == s.eos)
        if fin:
            s.status = Sequence.FINISHED
            self.running.remove(s)
            self.alloc.free(s.blocks)
            s.blocks = []
            self.done[s.id] = s
        return fin

    def step(self):
        """One iteration.  Returns [(request id, new token, finished)] for every sequence that produced a token."""
        decode, prefill = self._schedule()
        seqs = decode + [s for s, _ in prefill]
        if not seqs:
            if self.waiting and not self.running:
                raise MemoryError("the KV-cache pool cannot hold the next waiting request")
            return []
        if self.num_speculative_tokens:
            return self._speculative_step(decode, prefill)
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
            out.append((s.id, tok, self._finish_token(s, tok)))
        self.stats["max_running"] = max(self.stats["max_running"], len(self.running))
        return out

    # ---- speculative decoding -----------------------------------------------------------------------------------------------------
    def _propose(self, spec, prefill):
        """Draft phase: {sequence: its s.spec proposed tokens}.  The first draft forward carries every token the draft's cache lacks up to
        where the target's cache will be after this step (greedy prefill chunks, and each speculating row's last token); then k_s - 1
        single-token forwards, a sequence dropping out once it has its k_s proposals."""
        ends = [(s, s.cached + 1) for s in spec] + [(s, s.cached + n) for s, n in prefill if not s.do_sample]
        seqs = [s for s, _ in ends]
        n_new = [e - s.draft_cached for s, e in ends]
        if not seqs:
            return {}
        logits = self._run(self._draft, seqs, n_new, [n if s.draft_cached == 0 else 0 for s, n in zip(seqs, n_new)],
                           [s.draft_cached for s in seqs])
        for s, n in zip(seqs, n_new):
            s.draft_cached += n
        prop = {s: [int(t)] for s, t in zip(spec, logits[:len(spec)].argmax(-1).tolist())}
        for i in range(1, max((s.spec for s in spec), default=0)):
            act = [s for s in spec if s.spec > i]
            start = [s.draft_cached for s in act]
            logits = self._run(self._draft, act, [1] * len(act), [0] * len(act), start, [[prop[s][-1]] for s in act])
            for s, t in zip(act, logits.argmax(-1).tolist()):
                s.draft_cached += 1
                prop[s].append(int(t))
        return prop

    def _speculative_step(self, decode, prefill):
        spec = [s for s in decode if s.spec > 0]
        prop = self._propose(spec, prefill)
        seqs = decode + [s for s, _ in prefill]
        n_new = [1 + s.spec for s in decode] + [n for _, n in prefill]
        enc = [0] * len(decode) + [n if s.cached == 0 else 0 for s, n in prefill]
        dec = [s.cached for s in seqs]
        toks = [[s.tokens()[s.cached]] + prop.get(s, []) for s in decode] + [s.tokens()[s.cached:s.cached + n] for s, n in prefill]
        ends = [sum(n_new[:i + 1]) for i in range(len(seqs))]
        rows = [r for s, n, e in zip(decode, n_new, ends) for r in range(e - n, e)] + [e - 1 for e in ends[len(decode):]]
        logits = self._run(self._target, seqs, n_new, enc, dec, toks, rows)      # every verify row, each prefill row's last
        self.stats["steps"] += 1
        self.stats["prefill_tokens"] += sum(n_new[len(decode):])
        out, r = [], 0
        for s in decode:
            k = s.spec
            if k == 0:
                emit = [int(_sample(logits[r: r + 1], s.do_sample, s.temperature, s.top_k, s.top_p)[0])]
            else:
                best = logits[r: r + k + 1].argmax(-1).tolist()
                a = 0
                while a < k and prop[s][a] == best[a]:
                    a += 1
                emit = prop[s][:a] + [int(best[a])]
                self.stats["draft_tokens"] += k
                self.stats["accepted_tokens"] += a
            r += k + 1
            s.cached += len(emit)               # the last token and the accepted proposals are now in the target's cache
            s.draft_cached = min(s.draft_cached, s.cached)
            for tok in emit:
                fin = self._finish_token(s, tok)
                out.append((s.id, tok, fin))
                self.stats["decode_tokens"] += 1
                if fin:
                    break
            else:                               # blocks reserved for rejected proposals go back to the pool
                keep = self._blocks_for(s.cached + 1)
                self.alloc.free(s.blocks[keep:])
                del s.blocks[keep:]
        for s, n in prefill:
            i = r
            r += 1
            s.cached += n
            if s.status != Sequence.RUNNING:
                s.status = Sequence.RUNNING
                self.running.append(s)
            if s.cached < s.target:
                continue
            tok = int(_sample(logits[i: i + 1], s.do_sample, s.temperature, s.top_k, s.top_p)[0])
            out.append((s.id, tok, self._finish_token(s, tok)))
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
