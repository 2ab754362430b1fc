"""block_multihead_attention's qkv prologue fused into the paged cache write (csrc/kv_cache_quant.cu, `paged_kv_cache_write` with qkv_out /
qkv_out_scale / qkv_bias / rope) and its output quantization (`attention_out_quant`) on the GPU: mixed batches against the reference on the
same device, int32 against the float path, the output rule, launch accounting, the rope range check, and the compiled kernels."""
import hashlib
import json
import os
import re
import subprocess

import pytest
import torch

from paddle_b200 import kernels
from paddle_b200.incubate.nn import paged_attention as PA
from test_block_attention_prologue_cpu import _bits, mixed_batch, rope_emb_from_tables
from test_kv_cache_quant_gpu import _quantize_cache
from test_paged_prefill_gpu import _ext, rel_err
from test_prefix_caching_gpu import _shared_batch

pytestmark = pytest.mark.gpu

D = 128
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOUND = {torch.int8: 127.0, torch.float8_e4m3fn: 448.0}
# a fresh prompt, a continuing chunk longer than VERIFY_MAX, verify rows and plain decode rows beside one shared-prefix group
OTHERS = [(150, 0, 150), (0, 100, 40), (0, 63, 4), (0, 7, 1), (0, 500, 1)]


def _raw(t):
    return t.as_subclass(torch.Tensor)


def _mixed(nh, nkv, dtype, kv, seed):
    bs = 64
    qkv, kc, vc, args, sp = _shared_batch([(4 * bs, [3, 1, 20, 7])], OTHERS, nh, nkv, bs, dtype, seed=seed)
    quant = {}
    if kv is not None:
        bound = BOUND[kv]
        qs = torch.full((nkv,), 0.25, device="cuda")
        kc, vc = _quantize_cache(kc, kv, qs, bound, seed + 1), _quantize_cache(vc, kv, qs, bound, seed + 2)
        quant = dict(cache_k_quant_scales=qs, cache_v_quant_scales=qs, cache_k_dequant_scales=1.0 / (bound * qs),
                     cache_v_dequant_scales=1.0 / (bound * qs), quant_max_bound=bound, quant_min_bound=-bound)
    return qkv, kc, vc, args, sp, quant


def _same_cache(a, b):
    a, b = _bits(_raw(a)), _bits(_raw(b))
    if a.is_floating_point():
        a, b = a.nan_to_num(7.0), b.nan_to_num(7.0)
    return torch.equal(a, b)


@pytest.mark.parametrize("heads", [(32, 8), (32, 32)])
@pytest.mark.parametrize("neox", [False, True])
@pytest.mark.parametrize("kv", [None, torch.int8, torch.float8_e4m3fn])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_mixed_batch_matches_the_reference(dtype, kv, neox, heads):
    nh, nkv = heads
    qkv, kc, vc, args, sp, quant = _mixed(nh, nkv, dtype, kv, seed=nh + nkv + (3 if neox else 0))
    g = torch.Generator(device="cuda").manual_seed(1)
    pro = dict(qkv_bias=(torch.randn(qkv.shape[1], generator=g, device="cuda") * 0.3).to(dtype), rope_emb=rope_emb_from_tables(1024, neox, "cuda"),
               use_neox_style=neox, **quant)
    out, q1, kc1, vc1 = PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args, shared_prefix=sp, **pro)
    ref, q2, kc2, vc2 = PA._block_attention_ref(qkv.clone(), kc.clone(), vc.clone(), *args, shared_prefix=sp, **pro)
    assert torch.equal(_raw(q1), _raw(q2)) and not torch.equal(_raw(q1), qkv)
    assert _same_cache(kc1, kc2) and _same_cache(vc1, vc2)
    o, r = _raw(out).float(), _raw(ref).float()
    assert torch.isfinite(o).all()
    cu = args[3].tolist()
    for b in range(len(cu) - 1):
        e = rel_err(o[cu[b]:cu[b + 1]], r[cu[b]:cu[b + 1]])
        assert e < 2e-2, (b, e)


@pytest.mark.parametrize("kv", [None, torch.int8])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_int32_qkv_is_bitwise_the_float_path(dtype, kv):
    nh, nkv = 32, 8
    qkv, kc, vc, args, sp, quant = _mixed(nh, nkv, dtype, kv, seed=9)
    g = torch.Generator(device="cuda").manual_seed(2)
    w = qkv.shape[1]
    qi = torch.randint(-3000, 3000, qkv.shape, generator=g, device="cuda", dtype=torch.int32)
    col_scale = torch.rand(w, generator=g, device="cuda") * 4e-4
    pro = dict(qkv_bias=(torch.randn(w, generator=g, device="cuda") * 0.2).to(dtype), rope_emb=rope_emb_from_tables(1024, False, "cuda"), **quant)
    got = PA.block_attention(qi.clone(), kc.clone(), vc.clone(), *args, shared_prefix=sp, qkv_out_scale=col_scale,
                             compute_dtype="bf16" if dtype == torch.bfloat16 else "fp16", **pro)
    rows = (qi.float() * col_scale).to(dtype)
    want = PA.block_attention(rows, kc.clone(), vc.clone(), *args, shared_prefix=sp, **pro)
    assert torch.equal(_raw(got[1]), qi)
    assert torch.equal(_raw(got[0]), _raw(want[0]))
    assert _same_cache(got[2], want[2]) and _same_cache(got[3], want[3])


@pytest.mark.parametrize("out_kind", ["int8_rne", "int8_away", "int8_shift", "fp8", "int8_no_prologue"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_out_scale_is_bitwise_the_rule_on_the_16bit_output(dtype, out_kind):
    nh, nkv = 32, 8
    qkv, kc, vc, args, sp, _ = _mixed(nh, nkv, dtype, None, seed=11)
    g = torch.Generator(device="cuda").manual_seed(3)
    kw = dict(rope_emb=rope_emb_from_tables(1024, True, "cuda"), use_neox_style=True)
    if out_kind == "fp8":
        kw.update(quant_max_bound=448.0, quant_min_bound=-448.0)
    else:
        kw.update(quant_round_type=0 if out_kind == "int8_rne" else 1)
    if out_kind == "int8_no_prologue":                                         # out_scale alone: the fused write stores the rows as they are
        kw = {}
    if out_kind == "int8_shift":
        kw.update(out_shift=(torch.randn(nh * D, generator=g, device="cuda") * 0.1).to(dtype),
                  out_smooth=(torch.rand(nh * D, generator=g, device="cuda") + 0.5).to(dtype))
    o16 = _raw(PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args, shared_prefix=sp, out_scale=-1, **kw)[0])
    out_scale = 1.0 / 127.0 * 256.0                                          # many exact ties, and values beyond the bounds
    y = _raw(PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args, shared_prefix=sp, out_scale=out_scale, **kw)[0])
    pro = PA.qkv_prologue_params(qkv, nh, nkv, D, out_scale=out_scale, **{k: v for k, v in kw.items() if k not in ("rope_emb", "use_neox_style")})
    want = PA._out_quant_ref(o16, pro)
    assert y.dtype == want.dtype == (torch.float8_e4m3fn if out_kind == "fp8" else torch.int8)
    assert torch.equal(_bits(y), _bits(want))
    if out_kind != "fp8":
        assert (y == 127).any() and (y == -127).any()


def test_launch_accounting(monkeypatch):
    nh, nkv = 32, 8
    qkv, kc, vc, args, _ = mixed_batch([(300, 0, 300), (0, 64, 100)], nh, nkv, 64, torch.bfloat16, seed=4, device="cuda")
    kernels.reset_launch_count()
    PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args)       # 16-bit cache, no prologue: a torch scatter and the attention
    attention = kernels.launch_count()
    writes = []
    real_write = _ext().paged_kv_cache_write

    def write(*a, **k):
        writes.append(k)
        return real_write(*a, **k)

    def boom(*a, **k):
        raise AssertionError("unexpected call beside the fused prologue")

    kw = dict(qkv_bias=torch.ones(qkv.shape[1], dtype=torch.bfloat16, device="cuda"), rope_emb=rope_emb_from_tables(512, False, "cuda"))
    monkeypatch.setattr(_ext(), "paged_kv_cache_write", write)
    monkeypatch.setattr(PA, "_block_attention_ref", boom)
    monkeypatch.setattr(torch, "bucketize", boom)                            # the 16-bit scatter's first step
    kernels.reset_launch_count()
    out = PA.block_attention(qkv.clone(), kc, vc, *args, **kw)[0]
    assert kernels.launch_count() == attention + 1 and len(writes) == 1       # the cache write is the one fused launch
    assert writes[0]["qkv_bias"] is not None and writes[0]["rope_cos"] is not None
    assert torch.isfinite(_raw(out).float()).all()
    kernels.reset_launch_count()
    out = PA.block_attention(qkv.clone(), kc, vc, *args, out_scale=0.5, **kw)[0]
    assert kernels.launch_count() == attention + 2 and len(writes) == 2 and _raw(out).dtype == torch.int8


def test_rope_position_past_the_table_raises_before_any_launch():
    qkv, kc, vc, args, _ = mixed_batch([(20, 0, 20), (0, 70, 1)], 8, 2, 16, torch.bfloat16, seed=5, device="cuda")
    k0, v0 = kc.clone(), vc.clone()
    kernels.reset_launch_count()
    with pytest.raises(ValueError, match="position 70"):
        PA.block_attention(qkv, kc, vc, *args, rope_emb=rope_emb_from_tables(70, False, "cuda"))
    assert kernels.launch_count() == 0
    assert torch.equal(kc, k0) and torch.equal(vc, v0)


def _sass_functions():
    obj = os.path.join(ROOT, "paddle_b200", "_build_cache", "kv_cache_quant.cuda.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = f.split("\n", 1)
        out[name.strip()] = [re.sub(r"/\*[0-9a-f]{4}\*/", "", ln).strip() for ln in body.split("\n") if re.search(r"/\*[0-9a-f]{4}\*/", ln)]
    return out


def test_cache_write_kernels_sass():
    funcs = _sass_functions()
    new = [n for n in funcs if "prologue_write_kernel" in n or "out_quant_kernel" in n]
    assert len(new) == 2 * 2 * 3 * 3 + 2 * 2                                  # T x input x cache x rope, and T x output format
    for n in new:
        assert not any(re.search(r"\b(LDL|STL)\b", ins) for ins in funcs[n]), n
    # the plain 8-bit write compiles to the instructions it compiled to before the prologue was added
    with open(os.path.join(ROOT, "tests", "golden", "kv_cache_write_sass.json")) as f:
        golden = json.load(f)
    old = {n: hashlib.sha256("\n".join(ins).encode()).hexdigest() for n, ins in funcs.items() if "cache_write_kernel" in n}
    assert old == golden
