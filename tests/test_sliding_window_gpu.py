"""Sliding-window attention on the GPU: the windowed decode, verify and prefill kernels against the reference in mixed batches (16- and
8-bit caches, head_dim 128 and 64, block sizes 16 - 256, three head layouts, NaN in every out-of-window block and unused row), bit-equality
with the unwindowed kernels when the window covers every context, generate()'s windowed decode kernel against the model forward, LLMEngine
on a windowed model against generate(), and the windowed model's training forward and backward on the column-mask kernels (needs a GPU)."""
import math

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import kernels, models
from paddle_b200.framework.flags import set_flags
from paddle_b200.incubate.nn import paged_attention as PA

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _raw(t):
    return t.as_subclass(torch.Tensor)


# (enc, dec, now): decode rows, a fresh prompt, continuing chunks, verify rows and empty rows around the window
SPECS = [(0, 7, 1), (0, 300, 1), (0, 2000, 1), (300, 0, 300), (0, 129, 200), (0, 1500, 400), (0, 50, 0), (0, 64, 3), (0, 999, 5),
         (0, 2100, 8), (0, 40, 2)]


def _batch(specs, nh, nkv, d, bs, dtype, window, kv=None, seed=0):
    """Shuffled block tables.  Every cache row that holds no cached token, and every block wholly below a sequence's window, holds NaN
    (int8: +127); the table entries of the blocks below the window point at spare NaN blocks, as after a release and reuse."""
    g = torch.Generator().manual_seed(seed)
    now = torch.tensor([s[2] for s in specs], dtype=torch.int32)
    cu = torch.zeros(len(specs) + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(now, 0)
    need = [((0 if e > 0 else dd) + n + bs - 1) // bs for e, dd, n in specs]
    max_blocks, nblocks = max(need) + 2, sum(need) + 8
    perm = torch.randperm(nblocks, generator=g)
    spare = perm[sum(need):]
    bt = spare[torch.randint(0, spare.numel(), (len(specs), max_blocks), generator=g)].to(torch.int32)
    cdt = dtype if kv is None else kv
    fill = 127 if cdt == torch.int8 else float("nan")
    kc = torch.full((nblocks, nkv, bs, d), fill, dtype=cdt)
    vc = torch.full_like(kc, fill)
    nxt = 0
    for b, (e, dd, n) in enumerate(specs):
        bt[b, :need[b]] = perm[nxt:nxt + need[b]].to(torch.int32)
        nxt += need[b]
        past = 0 if e > 0 else dd
        lo = max(0, past - window + 1)                          # the lowest key any new token of the sequence sees
        pos = torch.arange(lo, past)
        blk = bt[b].long()[pos // bs]
        if kv == torch.int8:
            kc[blk, :, pos % bs] = torch.randint(-100, 100, (pos.numel(), nkv, d), generator=g, dtype=torch.int8)
            vc[blk, :, pos % bs] = torch.randint(-100, 100, (pos.numel(), nkv, d), generator=g, dtype=torch.int8)
        else:
            kc[blk, :, pos % bs] = (torch.randn(pos.numel(), nkv, d, generator=g) * 0.5).to(cdt)
            vc[blk, :, pos % bs] = (torch.randn(pos.numel(), nkv, d, generator=g) * 0.5).to(cdt)
        dead = lo // bs                                          # blocks wholly below the window: handed to "another sequence"
        bt[b, :dead] = spare[torch.randint(0, spare.numel(), (dead,), generator=g)].to(torch.int32)
    qkv = (torch.randn(int(cu[-1]), (nh + 2 * nkv) * d, generator=g) * 0.5).to(dtype)
    enc = torch.tensor([s[0] for s in specs], dtype=torch.int32)
    dec = torch.tensor([s[1] for s in specs], dtype=torch.int32)
    args = (enc.cuda(), dec.cuda(), now.cuda(), cu.cuda(), bt.cuda(), bs)
    quant = {}
    if kv is not None:
        bound = 127.0 if kv == torch.int8 else 448.0
        dq = (2.0 ** -torch.randint(5, 9, (nkv,), generator=g).float()).cuda()
        quant = dict(cache_k_quant_scales=1.0 / (dq * bound), cache_v_quant_scales=1.0 / (dq * bound), cache_k_dequant_scales=dq,
                     cache_v_dequant_scales=dq, quant_max_bound=bound, quant_min_bound=-bound)
    return qkv.cuda(), kc.cuda(), vc.cuda(), args, quant


def _check(specs, nh, nkv, d, bs, dtype, window, kv=None):
    qkv, kc0, vc0, args, quant = _batch(specs, nh, nkv, d, bs, dtype, window, kv)
    kernels.reset_launch_count()
    out, _, _, _ = PA.block_attention(qkv, kc0.clone(), vc0.clone(), *args, **quant, sliding_window=window)
    assert kernels.launch_count() >= 6                          # decode, verify and prefill: two launches each
    ref, _, _, _ = PA._block_attention_ref(qkv, kc0.clone(), vc0.clone(), *args, **quant, sliding_window=window)
    o, r = _raw(out).float(), _raw(ref).float()
    assert torch.isfinite(o).all()
    cu = args[3].tolist()
    for b in range(len(specs)):
        e = rel_err(o[cu[b]:cu[b + 1]], r[cu[b]:cu[b + 1]]) if cu[b + 1] > cu[b] else 0.0
        assert e < 2e-2, (b, specs[b], e)


@pytest.mark.parametrize("window", [1, 100, 1000])
@pytest.mark.parametrize("heads", [(32, 4), (8, 8), (16, 2)])
@pytest.mark.parametrize("bs", [16, 64, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_windowed_kernels_match_reference(dtype, bs, heads, window):
    _check(SPECS, *heads, 128, bs, dtype, window)


@pytest.mark.parametrize("window", [7, 200])
@pytest.mark.parametrize("bs", [32, 128])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_windowed_kernels_head_dim_64(dtype, bs, window):
    _check(SPECS, 16, 2, 64, bs, dtype, window)


@pytest.mark.parametrize("kv", [torch.int8, torch.float8_e4m3fn])
@pytest.mark.parametrize("bs", [16, 64, 256])
def test_windowed_kernels_8bit_caches(kv, bs):
    _check(SPECS, 8, 2, 128, bs, torch.bfloat16, 333, kv)


@pytest.mark.parametrize("d,kv", [(128, None), (64, None), (128, torch.int8)])
def test_window_covering_the_context_is_bit_equal_to_no_window(d, kv):
    qkv, kc, vc, args, quant = _batch(SPECS, 16, 4, d, 64, torch.bfloat16, 10 ** 6, kv)
    a = _raw(PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args, **quant, sliding_window=10 ** 6)[0])
    b = _raw(PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args, **quant)[0])
    assert torch.equal(a, b)


def _tiny(window, seed=0, **kw):
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(seed)
        base = dict(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2, vocab_size=512,
                    max_position_embeddings=1024, sliding_window=window)
        base.update(kw)
        cfg = models.llama_tiny(**base)
        m = models.LlamaForCausalLM(cfg)
        m.eval()
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    return m, cfg


def test_generate_windowed_decode_kernel_matches_model_forward():
    m, cfg = _tiny(24)
    gen = models.LlamaGenerator(m)
    ids = torch.randint(1, cfg.vocab_size, (2, 40), generator=torch.Generator().manual_seed(0)).cuda()
    cache = models.KVCache(len(gen.layers), 2, gen.nkv, 64, gen.hd, torch.bfloat16, "cuda")
    set_flags({"FLAGS_b200_decode_kernel": True})
    try:
        with torch.no_grad():
            logits = gen.prefill(ids, torch.tensor([40, 40], device="cuda"), cache)
            seq = ids
            for _ in range(12):
                tok = logits.argmax(-1)
                seq = torch.cat([seq, tok[:, None]], 1)
                kernels.reset_launch_count()
                logits = gen.decode_step(tok, cache)
                assert kernels.launch_count() > 0
                full = _raw(m(seq))[:, -1].float()
                assert rel_err(logits.float(), full) < 3e-2
    finally:
        set_flags({"FLAGS_b200_decode_kernel": False})


def _alone(m, prompt, n):
    return _raw(models.generate(m, torch.tensor([prompt]).cuda(), max_new_tokens=n))[0, len(prompt):].tolist()


def _agrees(m, prompt, out, alone):
    """Greedy tokens `out` against generate()'s `alone`: equal up to the first difference, and from there on every token of `out` is the
    model forward's argmax up to a bf16 near-tie (random tiny models have many), so a wrong cache row cannot pass."""
    assert len(out) == len(alone)
    with torch.no_grad():
        logits = _raw(m(torch.tensor([prompt + out[:-1]]).cuda()))[0, len(prompt) - 1:].float()
    top = logits.max(-1).values
    picked = logits[torch.arange(len(out)), torch.tensor(out).cuda()]
    assert ((top - picked) <= 2e-2 * logits.abs().amax(-1)).all(), (top - picked).tolist()
    return next((i for i, (a, b) in enumerate(zip(out, alone)) if a != b), len(out))


def _prompts(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]


@pytest.mark.parametrize("chunk", [None, 48])
def test_engine_on_a_windowed_model_matches_generate(chunk):
    m, cfg = _tiny(40)
    prompts = _prompts(cfg, (30, 150, 77, 210), seed=0)
    eng = models.LLMEngine(m, num_blocks=40, block_size=16, max_batch_tokens=512, max_prefill_chunk=chunk)
    log = []
    alloc = eng.alloc.alloc
    eng.alloc.alloc = lambda: log.append(alloc()) or log[-1]
    ids = [eng.add_request(p, 48) for p in prompts]
    res = eng.run_until_done()
    same = [_agrees(m, p, res[i], _alone(m, p, 48)) for i, p in zip(ids, prompts)]
    assert min(same) >= 16, same
    assert eng.stats["released_blocks"] > 0 and eng.stats["preemptions"] == 0
    assert len(log) > eng.alloc.num_blocks                      # released blocks were handed out again
    assert eng.alloc.num_free() == 40


def test_engine_windowed_int8_cache():
    m, cfg = _tiny(40)
    prompt = _prompts(cfg, (260,), seed=1)[0]
    absmax = models.calibrate_kv_cache(m, [prompt])
    logits = {}
    for dt in (None, "int8"):
        eng = models.LLMEngine(m, num_blocks=64, block_size=16, kv_cache_dtype=dt, kv_cache_absmax=None if dt is None else absmax)
        calls = []
        fwd = eng._forward
        eng._forward = lambda *a, _f=fwd, _c=calls: _c.append(_f(*a)) or _c[-1]
        eng.add_request(prompt, 20)
        eng.run_until_done()
        assert eng.stats["released_blocks"] > 0
        logits[dt] = torch.stack([c[0].float() for c in calls])
    assert torch.isfinite(logits["int8"]).all()
    assert rel_err(logits["int8"], logits[None]) < 3e-2


def test_engine_windowed_speculative_draft():
    m, cfg = _tiny(40)
    draft, _ = _tiny(40, seed=1, num_hidden_layers=1)
    prompts = _prompts(cfg, (70, 130), seed=2)
    eng = models.LLMEngine(m, num_blocks=48, block_size=16, draft_model=draft, num_speculative_tokens=3)
    ids = [eng.add_request(p, 40) for p in prompts]
    res = eng.run_until_done()
    for i, p in zip(ids, prompts):
        _agrees(m, p, res[i], _alone(m, p, 40))
    assert eng.stats["released_blocks"] > 0


def test_windowed_training_forward_backward_on_colmask_kernels():
    m, cfg = _tiny(48, num_key_value_heads=4)
    m.train()
    ids = torch.randint(0, cfg.vocab_size, (2, 257), generator=torch.Generator().manual_seed(0)).cuda()
    grads = {}
    for fused in (True, False):
        set_flags({"FLAGS_b200_flash_attention": fused})
        try:
            m.clear_gradients() if hasattr(m, "clear_gradients") else None
            for p in m.parameters():
                p.grad = None
            loss = m(ids[:, :-1], ids[:, 1:])
            loss.backward()
            grads[fused] = (float(loss), [_raw(p.grad).float().clone() for p in m.parameters() if p.grad is not None])
        finally:
            set_flags({"FLAGS_b200_flash_attention": True})
    assert abs(grads[True][0] - grads[False][0]) < 2e-2 * abs(grads[False][0])
    for a, b in zip(grads[True][1], grads[False][1]):
        assert rel_err(a, b) < 5e-2
