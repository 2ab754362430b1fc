"""Quantized paged KV cache on the GPU: the int8 / fp8 cache write (csrc/kv_cache_quant.cu) bit for bit against the reference, decode and
prefill over 8-bit blocks against the reference and bit for bit against the 16-bit kernels on dequantized caches, and LLMEngine logits
with int8 / fp8 caches against a bf16 cache."""
import math

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import kernels, models
from paddle_b200.incubate.nn import paged_attention as PA
from test_paged_prefill_gpu import SPECS, _batch, _ext, rel_err

pytestmark = pytest.mark.gpu

D = 128
BOUND = {torch.int8: 127.0, torch.float8_e4m3fn: 448.0}


def _bits(t):
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t


def _quantize_cache(c16, kv, quant_scale, bound, seed):
    """8-bit copy of a 16-bit cache [nb, Hkv, bs, D] whose unused rows are NaN: used rows quantized with the reference rules (round half
    away from zero), unused rows random bytes (int8) or NaN 0x7F (fp8)."""
    q = PA.kv_quant_params(c16[:1].to(kv), c16[:1].to(kv), quant_scale, quant_scale, quant_scale, quant_scale, quant_max_bound=bound,
                           quant_min_bound=-bound)
    used = torch.isfinite(c16.float()).all(-1, keepdim=True)
    x = torch.nan_to_num(c16.float()).permute(0, 2, 1, 3)                     # [nb, bs, Hkv, D]: the head axis next to D
    c8 = PA.quantize_kv(x, quant_scale, q, kv).permute(0, 2, 1, 3).contiguous()
    g = torch.Generator(device=c16.device).manual_seed(seed)
    junk = (torch.randint(-128, 128, c8.shape, generator=g, device=c16.device, dtype=torch.int8) if kv == torch.int8
            else torch.full(c8.shape, 0x7F, dtype=torch.uint8, device=c16.device).view(kv))
    return torch.where(used, _bits(c8), _bits(junk)).view(kv).contiguous()


def _quant_batch(kv, nh, nkv, bs, dtype, round_type=1, seed=0):
    qkv, kc16, vc16, args = _batch(SPECS, nh, nkv, bs, dtype, seed=seed)
    bound = BOUND[kv]
    rows = qkv.float().reshape(qkv.shape[0], nh + 2 * nkv, D)
    kmax = torch.maximum(rows[:, nh:nh + nkv].abs().amax((0, 2)), torch.nan_to_num(kc16.float()).abs().amax((0, 2, 3)))
    vmax = torch.maximum(rows[:, nh + nkv:].abs().amax((0, 2)), torch.nan_to_num(vc16.float()).abs().amax((0, 2, 3)))
    quant = dict(cache_k_quant_scales=1.0 / kmax, cache_v_quant_scales=1.0 / vmax, cache_k_dequant_scales=kmax / bound,
                 cache_v_dequant_scales=vmax / bound, quant_round_type=round_type, quant_max_bound=bound, quant_min_bound=-bound)
    kc = _quantize_cache(kc16, kv, quant["cache_k_quant_scales"], bound, seed + 1)
    vc = _quantize_cache(vc16, kv, quant["cache_v_quant_scales"], bound, seed + 2)
    return qkv, kc, vc, args, quant


@pytest.mark.parametrize("kv,round_type", [(torch.int8, 0), (torch.int8, 1), (torch.float8_e4m3fn, 1)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_cache_write_is_bitwise_the_reference(kv, round_type, dtype):
    qkv, kc0, vc0, args, quant = _quant_batch(kv, 8, 2, 16, dtype, round_type)
    qkv = qkv * 1.5                                                          # some values beyond the calibrated absmax: clamped
    quant["cache_k_quant_scales"][0] = 32.0 / 127.0                          # 127 * scale is exactly 32: many exact ties in y
    _, _, kc1, vc1 = PA.block_attention(qkv, kc0.clone(), vc0.clone(), *args, **quant)
    _, _, kc2, vc2 = PA._block_attention_ref(qkv, kc0.clone(), vc0.clone(), *args, **quant)
    for c1, c2, c0 in ((kc1, kc2, kc0), (vc1, vc2, vc0)):
        c1, c2, c0 = _bits(c1.as_subclass(torch.Tensor)), _bits(c2.as_subclass(torch.Tensor)), _bits(c0)
        assert torch.equal(c1, c2)
        changed = (c1 != c0).any(-1)
        assert changed.any()
    enc, dec, now, cu, bt, bs = args
    written = torch.zeros(kc0.shape[0], kc0.shape[2], dtype=torch.bool, device="cuda")     # [block, row] holding a new token
    for b in range(len(SPECS)):
        past = 0 if int(enc[b]) > 0 else int(dec[b])
        for pos in range(past, past + int(now[b])):
            written[int(bt[b, pos // bs]), pos % bs] = True
    keep = ~written[:, None, :, None].expand_as(kc0)
    assert torch.equal(_bits(kc1.as_subclass(torch.Tensor))[keep], _bits(kc0)[keep])
    assert torch.equal(_bits(vc1.as_subclass(torch.Tensor))[keep], _bits(vc0)[keep])


@pytest.mark.parametrize("kv", [torch.int8, torch.float8_e4m3fn])
@pytest.mark.parametrize("heads", [(8, 2), (4, 4)])
@pytest.mark.parametrize("bs", [16, 64, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quantized_block_attention_matches_reference(dtype, bs, heads, kv):
    nh, nkv = heads
    qkv, kc0, vc0, args, quant = _quant_batch(kv, nh, nkv, bs, dtype)
    kernels.reset_launch_count()
    out, _, kc1, vc1 = PA.block_attention(qkv, kc0.clone(), vc0.clone(), *args, **quant)
    assert kernels.launch_count() >= 1 + 2 + 2                               # cache write, decode (split + merge), prefill (work list + attention)
    ref, _, kc2, vc2 = PA._block_attention_ref(qkv, kc0.clone(), vc0.clone(), *args, **quant)
    out, ref = out.as_subclass(torch.Tensor), ref.as_subclass(torch.Tensor)
    assert torch.isfinite(out.float()).all()
    assert torch.equal(_bits(kc1.as_subclass(torch.Tensor)), _bits(kc2.as_subclass(torch.Tensor)))
    cu = args[3].tolist()
    for b in range(len(SPECS)):
        e = rel_err(out[cu[b]:cu[b + 1]], ref[cu[b]:cu[b + 1]])
        assert e < 2e-2, (b, SPECS[b], e)


def test_quantized_cuda_path_never_calls_the_reference(monkeypatch):
    qkv, kc, vc, args, quant = _quant_batch(torch.float8_e4m3fn, 8, 2, 64, torch.bfloat16)

    def boom(*a, **k):
        raise AssertionError("the CUDA path fell back to the reference")

    monkeypatch.setattr(PA, "_block_attention_ref", boom)
    out, _, _, _ = PA.block_attention(qkv, kc, vc, *args, **quant)
    assert torch.isfinite(out.as_subclass(torch.Tensor).float()).all()


def _pow2_scales(nkv, seed):
    g = torch.Generator().manual_seed(seed)
    return (2.0 ** -torch.randint(5, 9, (nkv,), generator=g).float()).cuda()   # power-of-two dequant scales: folding them is exact


def _random_8bit(shape, kv, g):
    if kv == torch.int8:
        return torch.randint(-127, 128, shape, generator=g, device="cuda", dtype=torch.int8)
    return (torch.randn(shape, generator=g, device="cuda") * 64).clamp(-448, 448).to(kv)


@pytest.mark.parametrize("kv", [torch.int8, torch.float8_e4m3fn])
@pytest.mark.parametrize("bs", [16, 64, 256])
def test_quantized_paged_prefill_is_bitwise_the_16bit_kernel(bs, kv):
    """2048 new rows over a 6000-token prefix: the 8-bit kernel equals the bf16 paged kernel on a cache holding the dequantized values."""
    g = torch.Generator(device="cuda").manual_seed(0)
    nh, nkv, past, n = 8, 2, 6000, 2048
    total = past + n
    nblk = (total + bs - 1) // bs
    pool = nblk + 5
    bt = torch.randperm(pool, device="cuda", generator=g)[:nblk].to(torch.int32).reshape(1, -1).contiguous()
    kc8, vc8 = _random_8bit((pool, nkv, bs, D), kv, g), _random_8bit((pool, nkv, bs, D), kv, g)
    kdq, vdq = _pow2_scales(nkv, 1), _pow2_scales(nkv, 2)
    kc16 = (kc8.float() * kdq[None, :, None, None]).to(torch.bfloat16)
    vc16 = (vc8.float() * vdq[None, :, None, None]).to(torch.bfloat16)
    q = (torch.randn(n, nh, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    scale = 1.0 / math.sqrt(D)
    outs = []
    for kc, vc, dq in ((kc8, vc8, dict(k_dequant_scales=kdq, v_dequant_scales=vdq)), (kc16, vc16, {})):
        out = torch.zeros(n, nh * D, device="cuda", dtype=torch.bfloat16)
        lse = torch.zeros(nh, n, device="cuda", dtype=torch.float32)
        _ext().attention_fwd_paged(q, kc, vc, bt, i32(0), i32(n), i32(past), scale, out, lse, **dq)
        outs.append((out, lse))
    assert torch.isfinite(outs[0][0].float()).all()
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("kv", [torch.int8, torch.float8_e4m3fn])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quantized_decode_is_bitwise_the_16bit_kernel(dtype, kv):
    """The decode rows of the mixed batch: the 8-bit decode kernel equals the 16-bit one on the dequantized cache."""
    g = torch.Generator(device="cuda").manual_seed(0)
    nh, nkv, bs = 8, 2, 16
    lens = [int(d) + 1 for e, d, n in SPECS if n == 1 and e == 0]
    nblk = [(n + bs - 1) // bs for n in lens]
    pool = sum(nblk) + 4
    perm = torch.randperm(pool, device="cuda", generator=g).to(torch.int32)
    bt = torch.zeros(len(lens), max(nblk), dtype=torch.int32, device="cuda")
    o = 0
    for i, k in enumerate(nblk):
        bt[i, :k] = perm[o:o + k]
        o += k
    kc8, vc8 = _random_8bit((pool, nkv, bs, D), kv, g), _random_8bit((pool, nkv, bs, D), kv, g)
    kdq, vdq = _pow2_scales(nkv, 3), _pow2_scales(nkv, 4)
    kc16 = (kc8.float() * kdq[None, :, None, None]).to(dtype)
    vc16 = (vc8.float() * vdq[None, :, None, None]).to(dtype)
    q = (torch.randn(len(lens), nh, D, device="cuda", generator=g) * 0.5).to(dtype)
    L = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = 1.0 / math.sqrt(D)
    o8 = _ext().decode_attention_paged(q, kc8, vc8, L, bt, scale, k_dequant_scales=kdq, v_dequant_scales=vdq)
    o16 = _ext().decode_attention_paged(q, kc16, vc16, L, bt, scale)
    assert torch.isfinite(o8.float()).all()
    assert torch.equal(o8, o16)


@pytest.mark.parametrize("kv,tol", [("int8", 3e-2), ("float8_e4m3fn", 8e-2)])
def test_engine_logits_with_quantized_cache(kv, tol):
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.llama_tiny(hidden_size=256, intermediate_size=512, num_attention_heads=2, num_key_value_heads=2, num_hidden_layers=2,
                                vocab_size=512, max_position_embeddings=1024)
        m = models.LlamaForCausalLM(cfg)
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    g = torch.Generator().manual_seed(0)
    prompt = torch.randint(1, cfg.vocab_size, (300,), generator=g).tolist()
    absmax = models.calibrate_kv_cache(m, [prompt])
    logits = {}
    for dt in (None, kv):
        eng = models.LLMEngine(m, num_blocks=64, block_size=16, kv_cache_dtype=dt, kv_cache_absmax=None if dt is None else absmax)
        calls = []
        fwd = eng._forward
        eng._forward = lambda *a, _f=fwd, _c=calls: _c.append(_f(*a)) or _c[-1]
        eng.add_request(prompt, 2)
        eng.run_until_done()
        logits[dt] = torch.stack([c[0].float() for c in calls])       # the prompt's last position, then the decode step
    assert torch.isfinite(logits[kv]).all()
    assert rel_err(logits[kv], logits[None]) < tol
