"""models.LLMEngine(enable_prefix_caching=True): full KV blocks are registered under a chained key of their token ids, later requests (and
readmitted preempted ones) reuse them, and unreferenced registered blocks stay matchable until evicted in LRU order.  Greedy tokens equal
isolated generation in every case; the hit accounting, the block states and the shared_prefix contract of block_attention are checked."""
import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models
from paddle_b200.incubate.nn import paged_attention as PA
from paddle_b200.models.serving import PrefixCachingAllocator


def _model(seed=0, **kw):
    paddle.seed(seed)
    cfg = models.llama_tiny(**kw)
    m = models.LlamaForCausalLM(cfg)
    m.eval()
    return m, cfg


def _alone(m, prompt, n):
    out = models.generate(m, torch.tensor([prompt]), max_new_tokens=n).as_subclass(torch.Tensor)
    return out[0, len(prompt):].tolist()


def _rand(cfg, n, g):
    return torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist()


def _check_blocks(eng):
    """Every block is free, evictable, or referenced by exactly its refcount's number of running sequences."""
    a = eng.alloc
    holders = {}
    for s in eng.running:
        for b in s.blocks:
            holders[b] = holders.get(b, 0) + 1
    free, evict = set(a._free), set(a.evictable)
    assert len(free) == len(a._free) and not free & evict
    for b in range(a.num_blocks):
        states = (b in free) + (b in evict) + (b in a.ref)
        assert states == 1, b
        assert a.ref.get(b, 0) == holders.get(b, 0), b
        if b in evict:
            assert b in a.key_of
    assert all(a.table[k] == b for b, k in a.key_of.items()) and len(a.table) == len(a.key_of)


def _run(eng, check=True):
    while eng.has_unfinished():
        eng.step()
        if check:
            _check_blocks(eng)
    assert eng.alloc.num_free() == eng.alloc.num_blocks
    return {i: s.generated for i, s in eng.done.items()}


def test_shared_system_prompt_hits_and_counts():
    m, cfg = _model()
    g = torch.Generator().manual_seed(0)
    system = _rand(cfg, 10, g)                                        # 2 full blocks of 4 and a partial one
    prompts = [system + _rand(cfg, n, g) for n in (3, 5, 1, 6)]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, enable_prefix_caching=True)
    ids = [eng.add_request(prompts[0], 6)]
    eng.step()                                                        # the first prompt registers its full blocks
    ids += [eng.add_request(p, 6) for p in prompts[1:]]
    res = _run(eng)
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 6), i
    hits = 3 * 8
    assert eng.stats["prefix_hit_tokens"] == hits
    assert eng.stats["prefill_tokens"] == sum(len(p) for p in prompts) - hits


def test_identical_prompts_and_a_block_multiple():
    m, cfg = _model()
    g = torch.Generator().manual_seed(1)
    p = _rand(cfg, 8, g)                                              # exactly 2 blocks: only the first may be shared
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, enable_prefix_caching=True)
    a, b = eng.add_request(p, 5), eng.add_request(p, 5)               # admitted together: nothing registered yet, no hit
    eng.step()
    assert eng.stats["prefix_hit_tokens"] == 0
    sa, sb = eng.running
    assert sa.blocks[0] in eng.alloc.key_of and sb.blocks[0] not in eng.alloc.key_of   # the same key: the second block stays private
    c = eng.add_request(p, 5)
    eng.step()
    assert eng.stats["prefix_hit_tokens"] == 4                        # the last block is recomputed: its last token gives the logits
    sc = next(s for s in eng.running if s.id == c)
    assert sc.blocks[0] == sa.blocks[0]
    res = _run(eng)
    ref = _alone(m, p, 5)
    assert res[a] == res[b] == res[c] == ref
    assert eng.stats["prefill_tokens"] == 3 * 8 - 4


@pytest.mark.parametrize("chunk", [3, 7])
def test_mid_flight_arrivals_and_chunked_prefill(chunk):
    m, cfg = _model()
    g = torch.Generator().manual_seed(2)
    system = _rand(cfg, 13, g)
    prompts = [system + _rand(cfg, n, g) for n in (2, 9, 4, 1)] + [_rand(cfg, 11, g)]
    news = [6, 4, 8, 5, 7]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, max_batch_tokens=12, max_prefill_chunk=chunk, enable_prefix_caching=True)
    ids = [eng.add_request(prompts[0], news[0])]
    for _ in range(6):                                               # the first prompt is fully cached after ceil(15 / chunk) steps
        eng.step()
        _check_blocks(eng)
    ids.append(eng.add_request(prompts[1], news[1]))
    eng.step()
    ids += [eng.add_request(p, n) for p, n in zip(prompts[2:], news[2:])]
    res = _run(eng)
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n), i
    assert eng.stats["prefix_hit_tokens"] == 3 * 12
    assert eng.stats["prefill_tokens"] == sum(len(p) for p in prompts) - 3 * 12


def test_preempted_sequence_reuses_its_own_blocks():
    m, cfg = _model(seed=1)
    g = torch.Generator().manual_seed(1)
    prompts = [_rand(cfg, 9, g) for _ in range(3)]
    eng = models.LLMEngine(m, num_blocks=9, block_size=4, enable_prefix_caching=True)
    ids = [eng.add_request(p, 10) for p in prompts]
    res = _run(eng)
    assert eng.stats["preemptions"] >= 1 and eng.stats["prefix_hit_tokens"] > 0
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 10)
    # every hit is a preempted sequence's own blocks: nothing else is shared between these prompts
    assert eng.stats["prefill_tokens"] + eng.stats["prefix_hit_tokens"] >= sum(len(p) for p in prompts)


def test_eviction_drops_the_least_recently_used_prefix():
    m, cfg = _model()
    g = torch.Generator().manual_seed(3)
    p1, p2 = _rand(cfg, 9, g), _rand(cfg, 21, g)
    eng = models.LLMEngine(m, num_blocks=6, block_size=4, enable_prefix_caching=True)
    a = eng.add_request(p1, 3)
    _run(eng)
    assert len(eng.alloc.evictable) == 2                              # p1's two full blocks (positions 0-7) stay matchable
    b = eng.add_request(p2, 3)                                        # needs all six blocks: both of p1's are evicted
    _run(eng)
    assert eng.stats["prefix_hit_tokens"] == 0
    c = eng.add_request(p2[:16] + _rand(cfg, 2, g), 3)                # p2's first 4 blocks are still there
    _run(eng)
    assert eng.stats["prefix_hit_tokens"] == 16
    d = eng.add_request(p1[:8] + _rand(cfg, 3, g), 3)                 # p1's were evicted: a miss
    _run(eng)
    assert eng.stats["prefix_hit_tokens"] == 16
    for i in (a, b, c, d):
        s = eng.done[i]
        assert s.generated == _alone(m, s.prompt, 3), i


def test_allocator_order_and_states():
    a = PrefixCachingAllocator(4)
    got = [a.alloc() for _ in range(3)]
    assert got == [0, 1, 2]                                           # the same order as BlockAllocator
    k0 = a.register(0, models.serving.BlockKey(None, [1, 2]))
    k1 = a.register(1, models.serving.BlockKey(k0, [3, 4]))
    assert a.register(2, models.serving.BlockKey(None, [1, 2])) is k0 and 2 not in a.key_of   # taken: block 2 stays private
    a.free(got)
    assert list(a.evictable) == [1, 0] and a._free == [3, 2] and a.num_free() == 4           # tail first
    blocks, keys = a.match([1, 2, 3, 4, 5], 2)
    assert blocks == [0, 1] and keys == [k0, k1]
    assert a.match([1, 2, 3, 9], 2)[0] == [0]
    assert [a.alloc(), a.alloc(), a.alloc()] == [2, 3, 1]             # free blocks first, then the least recently used
    assert a.match([1, 2, 3, 4], 2)[0] == [0]
    with pytest.raises(MemoryError):
        a.alloc(), a.alloc()


@pytest.mark.parametrize("kv", ["int8", "float8_e4m3fn"])
def test_quantized_caches(kv):
    m, cfg = _model()
    g = torch.Generator().manual_seed(4)
    system = _rand(cfg, 9, g)
    prompts = [system + _rand(cfg, n, g) for n in (3, 6, 2)]
    kw = dict(num_blocks=64, block_size=4, kv_cache_dtype=kv, kv_cache_absmax=models.calibrate_kv_cache(m, prompts))
    alone = []
    for p in prompts:
        e = models.LLMEngine(m, **kw)
        e.add_request(p, 6)
        alone.append(e.run_until_done()[0])
    eng = models.LLMEngine(m, enable_prefix_caching=True, **kw)
    ids = [eng.add_request(prompts[0], 6)]
    eng.step()
    ids += [eng.add_request(p, 6) for p in prompts[1:]]
    res = _run(eng)
    assert [res[i] for i in ids] == alone
    assert eng.stats["prefix_hit_tokens"] == 2 * 8


def test_draft_model_hits_set_draft_cached():
    m, cfg = _model()
    d, _ = _model(5, num_hidden_layers=1)
    g = torch.Generator().manual_seed(5)
    system = _rand(cfg, 11, g)
    prompts = [system + _rand(cfg, n, g) for n in (2, 5, 3)]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, draft_model=d, num_speculative_tokens=3, enable_prefix_caching=True)
    ids = [eng.add_request(prompts[0], 7)]
    eng.step()
    paddle.seed(9)
    ids.append(eng.add_request(prompts[1], 7))
    sampled = eng.add_request(prompts[2], 7, do_sample=True, temperature=0.8, top_k=20)
    eng.step()
    for s in eng.running:
        if s.id != ids[0]:
            assert s.cached >= 8 and s.draft_cached >= 8              # admitted with a hit of 8: both counts start there
    res = _run(eng)
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 7), i
    assert len(res[sampled]) == 7
    assert eng.stats["prefix_hit_tokens"] == 2 * 8


def test_sampling_request_blocks_do_not_register_with_a_draft():
    m, cfg = _model()
    g = torch.Generator().manual_seed(6)
    p = _rand(cfg, 10, g)
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, draft_model=m, num_speculative_tokens=2, enable_prefix_caching=True)
    eng.add_request(p, 5, do_sample=True)
    _run(eng)
    assert not eng.alloc.key_of
    eng.add_request(p, 5)
    _run(eng)
    assert eng.stats["prefix_hit_tokens"] == 0 and eng.alloc.key_of


def test_gpt_adapter():
    paddle.seed(6)
    cfg = models.gpt_tiny()
    m = models.GPTForCausalLM(cfg)
    m.eval()
    g = torch.Generator().manual_seed(7)
    system = _rand(cfg, 9, g)
    prompts = [system + _rand(cfg, n, g) for n in (4, 2, 6)]
    eng = models.LLMEngine(m, num_blocks=32, block_size=4, enable_prefix_caching=True)
    ids = [eng.add_request(prompts[0], 5)]
    eng.step()
    ids += [eng.add_request(p, 5) for p in prompts[1:]]
    res = _run(eng)
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 5)
    assert eng.stats["prefix_hit_tokens"] == 2 * 8


def test_sampling_requests_finish():
    m, cfg = _model()
    g = torch.Generator().manual_seed(8)
    system = _rand(cfg, 12, g)
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, enable_prefix_caching=True)
    paddle.seed(3)
    ids = [eng.add_request(system + _rand(cfg, n, g), 6, do_sample=True, temperature=0.9, top_k=20) for n in (1, 4)]
    eng.step()
    ids.append(eng.add_request(system + [5], 6, do_sample=True, top_p=0.9))
    res = _run(eng)
    assert all(len(res[i]) == 6 for i in ids)
    assert eng.stats["prefix_hit_tokens"] == 12


def test_caching_off_is_the_default_engine():
    m, cfg = _model()
    g = torch.Generator().manual_seed(9)
    system = _rand(cfg, 10, g)
    prompts = [system + _rand(cfg, n, g) for n in (3, 5)]
    runs = []
    for kw in ({}, dict(enable_prefix_caching=False)):
        eng = models.LLMEngine(m, num_blocks=32, block_size=4, **kw)
        ids = [eng.add_request(p, 6) for p in prompts]
        eng.step()
        blocks = [list(s.blocks) for s in eng.running]
        res = eng.run_until_done()
        runs.append(([res[i] for i in ids], dict(eng.stats), blocks, type(eng.alloc)))
    assert runs[0] == runs[1] and runs[0][3] is models.BlockAllocator


def test_decode_rows_grouped_through_the_reference(monkeypatch):
    """With the thresholds lowered, the engine passes shared_prefix groups every decode step; the reference checks their contract."""
    monkeypatch.setattr(PA, "SHARED_PREFIX_MIN_GROUP", 2)
    monkeypatch.setattr(PA, "SHARED_PREFIX_MIN_TOKENS", 4)
    m, cfg = _model(num_key_value_heads=2)
    g = torch.Generator().manual_seed(10)
    system = _rand(cfg, 9, g)
    prompts = [system + _rand(cfg, n, g) for n in (3, 5, 1, 4)]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, enable_prefix_caching=True)
    seen = []
    orig = eng._shared_prefix_groups
    eng._shared_prefix_groups = lambda *a: seen.append(orig(*a)) or seen[-1]
    ids = [eng.add_request(prompts[0], 8)]
    eng.step()
    ids += [eng.add_request(p, 8) for p in prompts[1:]]
    res = _run(eng)
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 8)
    groups = [s for s in seen if s is not None]
    assert groups and max(len(s[1]) for s in groups) == 4 and all(p % 4 == 0 and p >= 8 for s in groups for p in s[2])


def _ref_batch():
    """Three decode rows sharing block 0 (4 cached tokens each... 5, 6 and 7), one prefill row."""
    nh, nkv, d, bs = 2, 1, 128, 4
    g = torch.Generator().manual_seed(0)
    kc = torch.randn(16, nkv, bs, d, generator=g)
    vc = torch.randn(16, nkv, bs, d, generator=g)
    enc = torch.tensor([0, 0, 0, 3], dtype=torch.int32)
    dec = torch.tensor([5, 6, 7, 0], dtype=torch.int32)
    now = torch.tensor([1, 1, 1, 3], dtype=torch.int32)
    cu = torch.tensor([0, 1, 2, 3, 6], dtype=torch.int32)
    bt = torch.tensor([[0, 1, 9], [0, 2, 9], [0, 3, 9], [4, 9, 9]], dtype=torch.int32)
    qkv = torch.randn(6, (nh + 2 * nkv) * d, generator=g)
    return qkv, kc, vc, [enc, dec, now, cu, bt, bs]


def test_reference_checks_the_shared_prefix_contract():
    qkv, kc, vc, args = _ref_batch()
    plain = PA._block_attention_ref(qkv, kc.clone(), vc.clone(), *args)[0]
    grouped = PA._block_attention_ref(qkv, kc.clone(), vc.clone(), *args, shared_prefix=([0, 3], [0, 1, 2], [4]))[0]
    assert torch.equal(plain.as_subclass(torch.Tensor), grouped.as_subclass(torch.Tensor))
    t = lambda v: torch.tensor(v, dtype=torch.int32)                   # noqa: E731
    assert torch.equal(PA._block_attention_ref(qkv, kc.clone(), vc.clone(), *args, shared_prefix=(t([0, 2]), t([0, 2]), t([4])))[0]
                       .as_subclass(torch.Tensor)[[0, 2]], plain.as_subclass(torch.Tensor)[[0, 2]])
    bad = [
        ([0, 2], [0, 1, 2], [4]),          # cu_groups does not end at len(group_seqs)
        ([0, 0, 3], [0, 1, 2], [4, 4]),    # an empty group
        ([1, 3], [0, 1], [4]),             # cu_groups does not start at 0
        ([0, 2, 3], [0, 1, 1], [4, 4]),    # a sequence in two groups
        ([0, 2], [0, 7], [4]),             # not a batch index
        ([0, 2], [0, 1], [6]),             # not a multiple of block_size
        ([0, 2], [0, 1], [0]),             # not positive
        ([0, 2], [0, 3], [4]),             # a prefill row
        ([0, 2], [0, 1], [8]),             # the tables differ in block 1
        ([0, 3], [0, 1, 2], [4, 4]),       # prefix_len of the wrong length
        ([0, 2], [0, 1], [12]),            # past both sequences' cached tokens
        ([0, 2], [0, 1]),                  # not a triple
    ]
    for sp in bad:
        with pytest.raises(ValueError):
            PA._block_attention_ref(qkv, kc.clone(), vc.clone(), *args, shared_prefix=sp)
    args2 = list(args)
    args2[1] = torch.tensor([3, 6, 7, 0], dtype=torch.int32)          # sequence 0 has only 3 cached tokens: a 4-token prefix is too long
    with pytest.raises(ValueError):
        PA._block_attention_ref(qkv, kc.clone(), vc.clone(), *args2, shared_prefix=([0, 3], [0, 1, 2], [4]))
    with pytest.raises(ValueError):                                   # CUDA-less block_attention takes the reference and its checks
        PA.block_attention(qkv, kc.clone(), vc.clone(), *args, shared_prefix=([0, 2], [0, 3], [4]))
