"""Continuous-batching generation engine over a paged KV cache.

Role parity: the serving stack the reference assembles from `block_multihead_attention` (paged KV cache + block tables,
paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu) and its in-flight batching scheduler: requests join and leave the
running batch between steps, the KV cache is a pool of fixed-size blocks handed out on demand, and a sequence that cannot get a block is
preempted (its blocks go back to the pool; it is re-prefilled later from prompt + generated tokens).

Every step packs the tokens of all scheduled sequences into ONE [tokens, hidden] batch: whole prompts for the sequences being prefilled,
one token for the sequences being decoded.  The decoder layers run on the packed batch with the model's own sublayers; attention is
`incubate.nn.paged_attention.block_attention` - on CUDA (head_dim 128 or 64, fp16 / bf16) one indexed scatter of the new K / V rows into the
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

Prefix caching (`enable_prefix_caching=True`, off by default): a memory policy - cached blocks stay resident until they are evicted.  A full
block is registered once all its positions are in the cache, under a BlockKey (the previous block's key, its token ids); prompt and
generated-token blocks alike, so a preempted sequence finds its own blocks when it is readmitted.  Admission matches the longest chain of
registered blocks covering tokens[:total - 1] (the last token is always computed: its logits give the first sample), so the first computed
position is a block boundary and no sequence ever writes into a shared block.  The sequence starts with cached = the matched tokens; its
prefill is an ordinary continuing chunk, charged only the unmatched tokens.  Blocks are reference-counted (PrefixCachingAllocator): a
registered block nobody holds is evictable - still matchable, in LRU order, a finished sequence's chain joining tail first - and alloc()
takes a free block before evicting one; num_free() counts both.  A key already registered by another block (identical prompts admitted in
one step) leaves the block private.  With a draft model a block registers only once both caches hold it (min(cached, draft_cached) >= its
end), and a sampling request's blocks never register, since the draft writes rows for greedy sequences only; a hit sets draft_cached =
cached.  Each step the plain decode rows are grouped by their first block id; a group's prefix is its members' longest common run of
leading block ids, and groups that `paged_attention.shared_prefix_pays` accepts run on `decode_attention_paged_shared`, which reads that
prefix once per tile of members.  stats gains prefix_hit_tokens.  Not covered: multi-level (tree) prefixes, grouping verify rows, parallel
sampling (n > 1) and copy-on-write of partial blocks.

Sliding-window models (`sliding_window` = W in the target's config): every block_attention call passes the window, so the windowed kernels
read only the last W positions of each query.  After each step (so between the chunks of a chunked prefill too) block j of a sequence with
`cached` = c positions is dead once (j + 1) * block_size <= c - W + 1: no later query of the sequence sees it.  Dead blocks go back to the
pool and their slots in the sequence's block list stay as placeholders (RELEASED), so table indices stay positions / block_size; the
kernels never read those table entries.  A sequence's footprint thus stops growing at about W tokens; admission still reserves the whole
prompt.  With a draft model the caches share block ids, so a block is released only when it is dead for the draft as well (a draft
without a window keeps every block of a greedy sequence).  stats gains released_blocks.  Not combinable with prefix caching.
"""
from __future__ import annotations

import torch

from ..incubate.nn.paged_attention import block_attention, shared_prefix_pays
from ..kernels import sampling
from .generation import _raw, _w


RELEASED = -1   # a sequence's block-list slot whose block went back to the pool (below its sliding window)


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


class BlockKey:
    """Identity of a full block's contents: the key of the block before it in its sequence (None for the first) and its block_size token
    ids.  The chain fixes the block's position, so equal keys mean equal K / V under static cache scales.  Equality compares token ids
    exactly (a hash collision never matches); the hash is computed once."""
    __slots__ = ("parent", "tokens", "_hash")

    def __init__(self, parent, tokens):
        self.parent, self.tokens = parent, tuple(tokens)
        self._hash = hash((None if parent is None else parent._hash, self.tokens))

    def __hash__(self):
        return self._hash

    def __eq__(self, other):
        return self is other or (isinstance(other, BlockKey) and self._hash == other._hash and self.tokens == other.tokens
                                 and self.parent == other.parent)


class PrefixCachingAllocator(BlockAllocator):
    """BlockAllocator with reference counts and a table of registered full blocks (LLMEngine(enable_prefix_caching=True)).

    A block is free, evictable (registered, no reference: still matchable, in LRU order) or referenced.  free() drops one reference per
    block; a registered block that reaches zero becomes the most recently used evictable block, any other goes back to the free list.
    alloc() takes a free block first, then evicts the least recently used evictable one (its key is dropped).  num_free() counts free plus
    evictable blocks: both can be handed out."""

    def __init__(self, num_blocks):
        super().__init__(num_blocks)
        self.ref = {}                  # block -> number of sequences holding it
        self.key_of = {}               # registered block -> its BlockKey
        self.table = {}                # BlockKey -> registered block
        self.evictable = {}            # registered blocks without a reference, least recently used first (dicts keep insertion order)

    def num_free(self):
        return len(self._free) + len(self.evictable)

    def alloc(self):
        if self._free:
            blk = self._free.pop()
        elif self.evictable:
            blk = next(iter(self.evictable))
            del self.evictable[blk]
            del self.table[self.key_of.pop(blk)]
        else:
            raise MemoryError("KV-cache block pool is exhausted")
        self.ref[blk] = 1
        return blk

    def free(self, blocks):
        for blk in reversed(blocks):  # tail first: a chain's end becomes evictable before its start
            self.ref[blk] -= 1
            if self.ref[blk] == 0:
                del self.ref[blk]
                if blk in self.key_of:
                    self.evictable[blk] = None
                else:
                    self._free.append(blk)

    def match(self, tokens, block_size):
        """(blocks, keys) of the longest chain of registered blocks that covers tokens[:k * block_size], k as large as possible."""
        blocks, keys, parent = [], [], None
        for j in range(len(tokens) // block_size):
            blk = self.table.get(BlockKey(parent, tokens[j * block_size:(j + 1) * block_size]))
            if blk is None:
                break
            parent = self.key_of[blk]            # the registered object: the next lookup compares parents by identity
            blocks.append(blk)
            keys.append(parent)
        return blocks, keys

    def acquire(self, blocks):
        """One more reference to each (registered) block; an evictable one leaves the eviction order."""
        for blk in blocks:
            self.evictable.pop(blk, None)
            self.ref[blk] = self.ref.get(blk, 0) + 1

    def register(self, blk, key):
        """Makes `blk` matchable under `key` and returns the registered key object, unless another block already holds the key: then
        `blk` stays private and that block's key is returned (children chain to it)."""
        have = self.table.get(key)
        if have is not None:
            return self.key_of[have]
        self.table[key], self.key_of[blk] = blk, key
        return key


class Sequence:
    WAITING, RUNNING, FINISHED = "waiting", "running", "finished"

    def __init__(self, seq_id, prompt, max_new_tokens, eos_token_id=None, do_sample=False, temperature=1.0, top_k=0, top_p=1.0, seed=0):
        self.id, self.prompt, self.max_new_tokens, self.eos = seq_id, [int(t) for t in prompt], int(max_new_tokens), eos_token_id
        self.do_sample, self.temperature, self.top_k, self.top_p, self.seed = do_sample, temperature, top_k, top_p, seed
        self.generated, self.blocks, self.cached, self.status, self.preemptions = [], [], 0, Sequence.WAITING, 0
        self.target = 0                            # tokens to prefill since admission: the sequence samples once cached reaches it
        self.draft_cached, self.spec = 0, 0        # speculative decoding: positions in the draft's cache, proposals this step
        self.keys = []                             # prefix caching: BlockKeys of the leading full blocks already keyed
        self.released = 0                          # sliding window: blocks[:released] went back to the pool (RELEASED slots)

    def owned(self):
        """The blocks the sequence holds (released slots excluded)."""
        return self.blocks[self.released:]

    def tokens(self):
        return self.prompt + self.generated

    def finished(self):
        return self.status == Sequence.FINISHED


_KV_CACHE_DTYPES = {"int8": (torch.int8, 127.0), "float8_e4m3fn": (torch.float8_e4m3fn, 448.0)}


class LLMEngine:
    """add_request() any time; step() runs one scheduler iteration (admit / preempt, one packed forward, one token per running sequence;
    with a draft model, up to num_speculative_tokens + 1 tokens per greedy decode sequence)."""

    def __init__(self, model, num_blocks=256, block_size=16, max_running=64, max_batch_tokens=8192, max_prefill_chunk=None, kv_cache_dtype=None,
                 kv_cache_absmax=None, draft_model=None, num_speculative_tokens=0, enable_prefix_caching=False):
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
        self.enable_prefix_caching = bool(enable_prefix_caching)
        self.alloc = PrefixCachingAllocator(num_blocks) if self.enable_prefix_caching else BlockAllocator(num_blocks)
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
        if self.enable_prefix_caching:
            self.stats["prefix_hit_tokens"] = 0
        self.window = getattr(self.cfg, "sliding_window", None)
        self._draft_window = getattr(self._draft[0].cfg, "sliding_window", None) if self._draft is not None else None
        if self.window is not None:
            if self.enable_prefix_caching:
                raise ValueError("enable_prefix_caching is not supported for a model with a sliding window")
            self.stats["released_blocks"] = 0

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
    def add_request(self, prompt_ids, max_new_tokens=32, eos_token_id=None, do_sample=False, temperature=1.0, top_k=0, top_p=1.0, seed=None):
        """Queues a request and returns its id.  A sampled request draws the token at position t (= len(prompt) + tokens generated so
        far) from Philox stream (seed, offset t), so with a `seed` its tokens depend only on its own logits: not on the requests that
        share its steps, preemption, chunked prefill or prefix-cache hits.  Without one it gets a seed from the default CPU generator
        here (paddle.seed makes a whole run reproducible)."""
        prompt = _raw(prompt_ids).reshape(-1).tolist() if isinstance(prompt_ids, torch.Tensor) else list(prompt_ids)
        need = (len(prompt) + max_new_tokens + self.block_size - 1) // self.block_size
        if need > self.alloc.num_blocks:
            raise ValueError(f"request needs {need} KV blocks, the pool has {self.alloc.num_blocks}")
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item()) if do_sample else 0
        seed = int(seed) & (2 ** 64 - 1)
        seed = seed - 2 ** 64 if seed >= 2 ** 63 else seed               # the same 64 bits as a signed int64
        s = Sequence(self._next_id, prompt, max_new_tokens, eos_token_id, do_sample, temperature, top_k, top_p, seed)
        self._next_id += 1
        self.waiting.append(s)
        return s.id

    def has_unfinished(self):
        return bool(self.waiting or self.running)

    # ---- scheduling -------------------------------------------------------------------------------------------------------------
    def _blocks_for(self, n_tokens):
        return (n_tokens + self.block_size - 1) // self.block_size

    def _preempt(self, s):
        self.alloc.free(s.owned())
        s.blocks, s.cached, s.draft_cached, s.status, s.keys, s.released = [], 0, 0, Sequence.WAITING, [], 0
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
            toks = s.tokens()
            total = len(toks)
            hits, keys = [], []
            if self.enable_prefix_caching:           # at least the last token is computed: its logits give the first sample
                hits, keys = self.alloc.match(toks[:total - 1], self.block_size)
            m = len(hits) * self.block_size
            n = total - m if chunk is None else min(chunk, total - m, budget)
            need = self._blocks_for(total + 1) - len(hits)
            held = sum(1 for b in hits if b in self.alloc.evictable) if hits else 0   # matched evictable blocks stop being available
            if n > budget or (chunk is not None and budget == 0) or need > self.alloc.num_free() - held:
                break
            self.waiting.pop(0)
            if hits:
                self.alloc.acquire(hits)
                self.stats["prefix_hit_tokens"] += m
            s.blocks = hits + [self.alloc.alloc() for _ in range(need)]
            s.keys, s.cached = keys, m
            if self.num_speculative_tokens:
                s.draft_cached = m                   # registered blocks hold their rows in both caches
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

    # ---- prefix caching -----------------------------------------------------------------------------------------------------------
    def _register(self, s, toks):
        """Keys and registers s's full blocks whose positions are all in the cache (with a draft: in both caches; a sampling request's
        draft cache is never written, so its blocks never register then).  toks: s's tokens, at least up to s.cached."""
        if not self.enable_prefix_caching or (self.num_speculative_tokens and s.do_sample):
            return
        end = min(s.cached, s.draft_cached) if self.num_speculative_tokens else s.cached
        bs = self.block_size
        for j in range(len(s.keys), end // bs):
            key = BlockKey(s.keys[-1] if s.keys else None, toks[j * bs:(j + 1) * bs])
            s.keys.append(self.alloc.register(s.blocks[j], key))

    def _shared_prefix_groups(self, seqs, n_new):
        """block_attention's shared_prefix argument for the plain decode rows among seqs (the first len(decode) of them, one new token and
        no speculation): rows are grouped by their first block id, a group's prefix is the longest run of leading block ids common to all
        its members, and only groups that paged_attention.shared_prefix_pays() accepts are passed.  None when there are none, and at
        head_dim 64, which has a decode kernel but no shared-prefix one: grouped rows would take block_attention's reference path."""
        if not self.enable_prefix_caching or self.hd == 64:
            return None
        by_first = {}
        for i, (s, n) in enumerate(zip(seqs, n_new)):
            if n == 1 and s.cached >= s.target and s.keys:     # a decode row with at least one registered (or shared) full block
                by_first.setdefault(s.blocks[0], []).append(i)
        cu, members, plen = [0], [], []
        for idx in by_first.values():
            if len(idx) < 2:
                continue
            first = seqs[idx[0]].blocks
            k = min(len(seqs[i].keys) for i in idx)
            for i in idx[1:]:
                b = seqs[i].blocks
                k = next((j for j in range(k) if b[j] != first[j]), k)
            if not shared_prefix_pays(len(idx), k * self.block_size, self.nh // self.nkv):
                continue
            members += idx
            cu.append(len(members))
            plen.append(k * self.block_size)
        return (cu, members, plen) if plen else None

    # ---- one packed forward -------------------------------------------------------------------------------------------------------
    def _forward(self, seqs, n_new, enc, dec):
        """The target model over this step's rows (s.tokens() from s.cached); logits of each sequence's last row [num_seqs, vocab]."""
        return self._run(self._target, seqs, n_new, enc, dec)

    @torch.no_grad()
    def _run(self, net, seqs, n_new, enc, dec, toks=None, rows=None):
        """One packed forward of `net` = (adapter, key caches, value caches, quantization args) over the sequences' blocks: n_new[i] tokens
        at positions dec[i] ... (toks[i], by default taken from s.tokens()).  Returns the logits of packed rows `rows` (default: each
        sequence's last row).  Target forwards pass the shared-prefix groups of their decode rows to block_attention."""
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
        shared = self._shared_prefix_groups(seqs, n_new) if net is self._target else None
        window = self.window if net is self._target else self._draft_window
        h = ad.embed_tokens(ids, position_ids)
        for li, layer in enumerate(ad.layers):
            qkv = ad.attn_in(layer, h, position_ids)
            t = qkv.shape[1]
            if self._observe is not None and net is self._target:
                self._observe(li, qkv.reshape(t, (nh + 2 * nkv) * hd))
            out, _, _, _ = block_attention(qkv.reshape(t, (nh + 2 * nkv) * hd), key_cache[li], value_cache[li], enc_t, dec_t, now_t, cu, bt,
                                           self.block_size, **kv_quant[li], shared_prefix=shared, sliding_window=window)
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
            self.alloc.free(s.owned())
            s.blocks, s.released = [], 0
            self.done[s.id] = s
        return fin

    def _release(self, s):
        """Sliding window: returns s's blocks that no later query of it can see to the pool (their slots become RELEASED)."""
        if self.window is None or s.status != Sequence.RUNNING:
            return
        end = s.cached - self.window + 1                         # the lowest key a query at position >= cached sees
        if self._draft is not None and not s.do_sample:          # the draft's cache uses the same block ids
            if self._draft_window is None:
                return
            end = min(end, s.draft_cached - self._draft_window + 1)
        dead = min(max(end, 0) // self.block_size, len(s.blocks))
        if dead > s.released:
            self.alloc.free(s.blocks[s.released:dead])
            self.stats["released_blocks"] += dead - s.released
            s.blocks[s.released:dead] = [RELEASED] * (dead - s.released)
            s.released = dead

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
        toks = self._sample_rows(logits, [s if s.cached + n >= s.target else None for s, n in zip(seqs, n_new)])
        out = []
        for i, (s, n) in enumerate(zip(seqs, n_new)):
            s.cached += n
            self._register(s, s.tokens())
            if s.status != Sequence.RUNNING:
                s.status = Sequence.RUNNING
                self.running.append(s)
            if s.cached < s.target:                # more chunks to come: nothing to sample yet
                continue
            tok = toks[i]
            out.append((s.id, tok, self._finish_token(s, tok)))
        for s in seqs:
            self._release(s)
        self.stats["max_running"] = max(self.stats["max_running"], len(self.running))
        return out

    def _sample_rows(self, logits, rows):
        """The next token of every logits row [len(rows), vocab] in one sampling call: rows[i] is the sequence row i samples for, or None
        for a greedy row (a verify row, or a prefill chunk that yields no token).  The per-row parameters go to the device as one packed
        copy and the ids come back as one copy."""
        n = len(rows)
        seed, offset, temp, top_p, top_k = [0] * n, [0] * n, [0.0] * n, [1.0] * n, [0] * n
        for i, s in enumerate(rows):
            if s is not None and s.do_sample and s.temperature != 0.0:
                seed[i], offset[i], temp[i] = s.seed, len(s.prompt) + len(s.generated), float(s.temperature)
                top_k[i] = min(max(int(s.top_k or 0), 0), 2 ** 31 - 1)
                top_p[i] = 1.0 if s.top_p is None else float(s.top_p)
        packed = torch.cat([torch.tensor([seed, offset], dtype=torch.int64).view(torch.uint8).reshape(-1),
                            torch.tensor([temp, top_p], dtype=torch.float32).view(torch.uint8).reshape(-1),
                            torch.tensor(top_k, dtype=torch.int32).view(torch.uint8).reshape(-1)]).to(self.device)
        i64 = packed[:16 * n].view(torch.int64)
        f32 = packed[16 * n:24 * n].view(torch.float32)
        ids = sampling.sample(logits, f32[:n], packed[24 * n:].view(torch.int32), f32[n:], i64[:n], i64[n:])[0]
        return ids.tolist()

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
        rows = [r for s in decode for r in ([s] if s.spec == 0 else [None] * (s.spec + 1))]
        toks = self._sample_rows(logits, rows + [s if s.cached + n >= s.target else None for s, n in prefill])
        out, r = [], 0
        for s in decode:
            k = s.spec
            if k == 0:
                emit = [toks[r]]
            else:
                best = toks[r: r + k + 1]                   # the target's argmax at every verify row
                a = 0
                while a < k and prop[s][a] == best[a]:
                    a += 1
                emit = prop[s][:a] + [int(best[a])]
                self.stats["draft_tokens"] += k
                self.stats["accepted_tokens"] += a
            r += k + 1
            s.cached += len(emit)               # the last token and the accepted proposals are now in the target's cache
            s.draft_cached = min(s.draft_cached, s.cached)
            self._register(s, s.tokens() + emit)
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
            self._register(s, s.tokens())
            if s.status != Sequence.RUNNING:
                s.status = Sequence.RUNNING
                self.running.append(s)
            if s.cached < s.target:
                continue
            tok = toks[i]
            out.append((s.id, tok, self._finish_token(s, tok)))
        for s in seqs:
            self._release(s)
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
