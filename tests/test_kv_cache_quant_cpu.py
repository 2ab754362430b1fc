"""Quantized paged KV cache (int8 / float8_e4m3fn) on the CPU path: the reference quantization rules, block_multihead_attention with
static cache scales, its argument checks, LLMEngine(kv_cache_dtype=...), and the compiled quantized kernels (registers, spills, wgmma
pipelining)."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models
from paddle_b200.incubate.nn import functional as IF
from paddle_b200.incubate.nn import paged_attention as PA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CACHE = os.path.join(ROOT, "paddle_b200", "_build_cache")


def _quant(dtype, round_type=1, bound=None):
    bound = bound if bound is not None else (127.0 if dtype == torch.int8 else 448.0)
    kc = torch.zeros(1, 1, 1, 1, dtype=dtype)
    one = torch.ones(1)
    return PA.kv_quant_params(kc, kc, one, one, one, one, quant_round_type=round_type, quant_max_bound=bound, quant_min_bound=-bound)


def _q(x, dtype, round_type=1, scale=1.0, bound=None):
    """quantize the values x (one head) with quant_scale = scale / bound, so y = scale * x (rounded in fp32 like the kernel)"""
    quant = _quant(dtype, round_type, bound)
    b = quant.max_bound
    qs = torch.tensor([scale], dtype=torch.float32) / b
    return PA.quantize_kv(torch.tensor(x, dtype=torch.float32).reshape(1, -1), qs, quant, dtype).reshape(-1)


def test_int8_round_half_to_even_and_away_from_zero():
    x = [0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 0.49999997, -0.49999997, 3.7, -3.2]
    # quant_scale 1 / 127 with bound 127: y = (127 * (1/127)) * x, and 127 * fl(1/127) is exactly 1 in fp32
    assert torch.tensor(127.0) * (torch.tensor(1.0) / 127.0) == 1.0
    assert _q(x, torch.int8, round_type=0).tolist() == [0, 0, 2, -2, 2, -2, 0, 0, 4, -3]
    assert _q(x, torch.int8, round_type=1).tolist() == [1, -1, 2, -2, 3, -3, 0, 0, 4, -3]


def test_int8_clamps_to_the_bounds():
    assert _q([300.0, -300.0, 126.6, -127.4], torch.int8).tolist() == [127, -127, 127, -127]
    assert _q([300.0, -300.0, 99.5, 1.0], torch.int8, bound=100.0).tolist() == [100, -100, 100, 1]


def test_fp8_rounds_to_nearest_even_like_torch():
    g = torch.Generator().manual_seed(0)
    x = torch.cat([torch.randn(4096, generator=g) * 100, torch.tensor([1000.0, -1000.0, 448.0, 0.0, 1.0625, 1.1875, 2 ** -10])])
    got = _q(x.tolist(), torch.float8_e4m3fn)
    want = x.clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
    assert got.float()[-7:-4].tolist() == [448.0, -448.0, 448.0]
    assert got.float()[-3:-1].tolist() == [1.0, 1.25]                 # ties between 1 and 1.125, 1.125 and 1.25: to the even mantissa


def _issue_example(dtype, quant):
    """2 heads, a 5-token prompt, block_size 16."""
    g = torch.Generator().manual_seed(0)
    nh = nkv = 2
    d, n, bs = 128, 5, 16
    qkv = torch.randn(n, (nh + 2 * nkv) * d, generator=g)
    kc = torch.zeros(4, nkv, bs, d, dtype=dtype)
    vc = torch.zeros_like(kc)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32)       # noqa: E731
    args = (i32(n), i32(0), i32(n), None, None, i32(0, n), None, torch.tensor([[2, 0]], dtype=torch.int32))
    out, _, kc, vc = IF.block_multihead_attention(qkv, kc, vc, *args, block_size=bs, **quant)
    return out.as_subclass(torch.Tensor), kc.as_subclass(torch.Tensor), qkv


@pytest.mark.parametrize("dtype,bound,tol", [(torch.int8, 127.0, 2e-2), (torch.float8_e4m3fn, 448.0, 6e-2)])
def test_block_multihead_attention_with_8bit_cache_is_within_quantization_error(dtype, bound, tol):
    ref, _, qkv = _issue_example(torch.float32, {})
    rows = qkv.reshape(5, 6, 128)
    amax = torch.stack([rows[:, 2:4].abs().amax(dim=(0, 2)), rows[:, 4:6].abs().amax(dim=(0, 2))])   # [2 (k, v), Hkv]
    quant = dict(cache_k_quant_scales=1.0 / amax[0], cache_v_quant_scales=1.0 / amax[1], cache_k_dequant_scales=amax[0] / bound,
                 cache_v_dequant_scales=amax[1] / bound, quant_max_bound=bound, quant_min_bound=-bound)
    out, kc, _ = _issue_example(dtype, quant)
    err = ((out - ref).norm() / ref.norm()).item()
    assert err < tol, err
    assert kc.dtype == dtype and kc[2, :, :5].float().abs().amax() > 0.5 * bound   # the cached rows use the 8-bit range


def test_quantization_argument_errors():
    one = torch.ones(2)
    scales = dict(cache_k_quant_scales=one, cache_v_quant_scales=one, cache_k_dequant_scales=one, cache_v_dequant_scales=one)
    with pytest.raises(NotImplementedError):
        _issue_example(torch.int8, dict(scales, use_dynamic_cachekv_quant=True))
    with pytest.raises(ValueError, match="16|float32|bfloat16|scales were given"):
        _issue_example(torch.float32, scales)
    with pytest.raises(ValueError, match="needs"):
        _issue_example(torch.int8, {})
    with pytest.raises(ValueError, match="needs"):
        _issue_example(torch.float8_e4m3fn, dict(cache_k_quant_scales=one))
    with pytest.raises(ValueError, match="448"):
        _issue_example(torch.float8_e4m3fn, dict(scales, quant_max_bound=500.0, quant_min_bound=-500.0))
    with pytest.raises(ValueError, match=r"\[H_kv\]"):
        _issue_example(torch.int8, dict(scales, cache_k_quant_scales=torch.ones(1, 2)))


# ---- LLMEngine with quantized caches ----------------------------------------------------------------------------------------------------
def _model(seed=0):
    paddle.seed(seed)
    cfg = models.llama_tiny()
    m = models.LlamaForCausalLM(cfg)
    m.eval()
    return m, cfg


def _prompts(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]


def _alone(m, kw, prompt, n):
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, **kw)
    i = eng.add_request(prompt, n)
    return eng.run_until_done()[i]


@pytest.mark.parametrize("kv", ["int8", "float8_e4m3fn"])
@pytest.mark.parametrize("chunk", [None, 3, 7])
def test_quantized_engine_batching_matches_serving_alone(kv, chunk):
    m, cfg = _model()
    prompts = _prompts(cfg, (5, 17, 9, 3, 22), seed=0)
    news = [6, 4, 8, 5, 3]
    kw = dict(kv_cache_dtype=kv, kv_cache_absmax=models.calibrate_kv_cache(m, prompts))
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, max_batch_tokens=12 if chunk else 64, max_prefill_chunk=chunk, **kw)
    assert eng.key_cache[0].dtype == getattr(torch, kv)
    ids = [eng.add_request(prompts[0], news[0]), eng.add_request(prompts[1], news[1])]
    eng.step()
    eng.step()
    ids.append(eng.add_request(prompts[2], news[2]))            # arrives mid-flight
    eng.step()
    ids += [eng.add_request(prompts[3], news[3]), eng.add_request(prompts[4], news[4])]
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, kw, p, n), i
    assert eng.alloc.num_free() == 64


@pytest.mark.parametrize("kv", ["int8", "float8_e4m3fn"])
def test_quantized_engine_with_preemption(kv):
    m, cfg = _model(seed=1)
    prompts = _prompts(cfg, (6, 11, 9), seed=1)
    kw = dict(kv_cache_dtype=kv, kv_cache_absmax=models.calibrate_kv_cache(m, prompts))
    eng = models.LLMEngine(m, num_blocks=9, block_size=4, max_batch_tokens=10, max_prefill_chunk=3, **kw)
    ids = [eng.add_request(p, 10) for p in prompts]
    res = eng.run_until_done()
    assert eng.stats["preemptions"] >= 1
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, kw, p, 10)


def test_engine_kv_cache_dtype_none_is_the_default():
    m, cfg = _model(seed=4)
    prompts = _prompts(cfg, (5, 17, 9, 3), seed=4)
    runs = []
    for kw in ({}, {"kv_cache_dtype": None}):
        eng = models.LLMEngine(m, num_blocks=12, block_size=4, max_batch_tokens=24, **kw)
        ids = [eng.add_request(p, 6) for p in prompts]
        res = eng.run_until_done()
        runs.append((dict(eng.stats), [res[i] for i in ids], eng.key_cache[0].dtype))
    assert runs[0] == runs[1]
    with pytest.raises(ValueError):
        models.LLMEngine(m, num_blocks=4, block_size=4, kv_cache_dtype="int8")                       # no absmax
    with pytest.raises(ValueError):
        models.LLMEngine(m, num_blocks=4, block_size=4, kv_cache_dtype="int4", kv_cache_absmax=torch.ones(2, 2, 2))


def test_calibration_covers_k_after_rotary_and_v():
    m, cfg = _model(seed=5)
    prompts = _prompts(cfg, (7, 12), seed=5)
    amax = models.calibrate_kv_cache(m, prompts)
    nkv = cfg.num_key_value_heads
    assert amax.shape == (cfg.num_hidden_layers, 2, nkv) and (amax > 0).all()
    eng = models.LLMEngine(m, num_blocks=16, block_size=4)
    seen = torch.zeros_like(amax)
    nh, hd = eng.nh, eng.hd

    def observe(li, qkv):
        r = qkv.reshape(qkv.shape[0], nh + 2 * nkv, hd).float()
        seen[li, 0] = torch.maximum(seen[li, 0], r[:, nh:nh + nkv].abs().amax(dim=(0, 2)))
        seen[li, 1] = torch.maximum(seen[li, 1], r[:, nh + nkv:].abs().amax(dim=(0, 2)))

    eng._observe = observe
    for p in prompts:
        eng.add_request(p, 1)
    eng.run_until_done()
    assert torch.equal(seen, amax)
    key_cache = eng.key_cache[0][:, :, :].float()      # what the 16-bit engine wrote into layer 0: the K rows after rotary
    assert key_cache.abs().amax(dim=(0, 2, 3)).le(amax[0, 0]).all()


# ---- the compiled kernels ----------------------------------------------------------------------------------------------------------------
_ATTN = os.path.join(CACHE, "attention_sm100.cuda.o")


@pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(_ATTN), reason="cuobjdump or the built objects are missing")
def test_quantized_prefill_kernels_are_pipelined_and_do_not_spill():
    out = subprocess.run(["cuobjdump", "-sass", _ATTN], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            res[name] = {"mma": 0, "arrive": 0, "local": 0}
        elif name is not None:
            res[name]["mma"] += bool(re.search(r"\b[HQI]GMMA\.", line))
            res[name]["arrive"] += "WARPGROUP.ARRIVE" in line
            res[name]["local"] += bool(re.search(r"\b(STL|LDL)\b", line))
    q8 = {k: v for k, v in res.items() if "4attn10fwd_kernel" in k and ("kv82I8" in k or "kv84E4M3" in k)}
    assert len(q8) == 4, sorted(res)
    for k, v in q8.items():
        assert 0 < v["arrive"] < v["mma"], (k, v)
        assert v["local"] == 0, (k, v)
