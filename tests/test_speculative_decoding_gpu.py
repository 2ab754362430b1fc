"""Multi-token paged decode (csrc/decode_attention.cu, `decode_attention_paged_multi`, behind block_attention's short continuing chunks)
against the reference in mixed batches, against successive single-token decode, its 8-bit instantiations bit for bit against the 16-bit
one, and LLMEngine's verify logits against plain decoding (needs a GPU)."""
import math
import os
import re
import subprocess

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import kernels, models
from paddle_b200.incubate.nn import paged_attention as PA
from test_kv_cache_quant_gpu import _pow2_scales, _random_8bit
from test_paged_prefill_gpu import _batch, _ext, rel_err

pytestmark = pytest.mark.gpu

D = 128
PASTS = (1, 5, 63, 64, 127, 1000, 6000)
NOWS = (2, 3, 5, 8, 16)


def _specs(nh, nkv):
    """Verify rows (every past x now within the row limit, longer ones too: they go to the prefill kernel), decode rows, long prefill."""
    g = nh // nkv
    ver = [(0, past, now) for past in PASTS for now in NOWS if now * g <= 64 or now == 16]
    return [(0, 7, 1), (300, 0, 300), (0, 129, 200)] + ver + [(0, 1000, 1)]


@pytest.mark.parametrize("heads", [(8, 2), (4, 4), (32, 4)])
@pytest.mark.parametrize("bs", [16, 64, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_mixed_batch_with_verify_rows_matches_reference(dtype, bs, heads):
    nh, nkv = heads
    specs = _specs(nh, nkv)
    qkv, kc0, vc0, args = _batch(specs, nh, nkv, bs, dtype)
    kernels.reset_launch_count()
    out, _, kc1, vc1 = PA.block_attention(qkv, kc0.clone(), vc0.clone(), *args)
    assert kernels.launch_count() >= 6                           # decode, multi-token decode and prefill: two launches each
    ref, _, kc2, vc2 = PA._block_attention_ref(qkv, kc0.clone(), vc0.clone(), *args)
    raw = lambda t: t.as_subclass(torch.Tensor)                  # noqa: E731
    assert torch.equal(raw(kc1).nan_to_num(7.0), raw(kc2).nan_to_num(7.0)) and torch.equal(raw(vc1).nan_to_num(7.0), raw(vc2).nan_to_num(7.0))
    o, r = raw(out).float(), raw(ref).float()
    assert torch.isfinite(o).all()
    cu = args[3].tolist()
    for b in range(len(specs)):
        e = rel_err(o[cu[b]:cu[b + 1]], r[cu[b]:cu[b + 1]])
        assert e < 2e-2, (b, specs[b], e)


def _cache(past, n, nkv, bs, dtype, g):
    total = past + n
    nblk = (total + bs - 1) // bs
    pool = nblk + 6
    perm = torch.randperm(pool, device="cuda", generator=g)
    bt = torch.cat([perm[:nblk], perm[nblk:nblk + 2]]).to(torch.int32).reshape(1, -1).contiguous()   # two NaN blocks past the end
    kc = torch.full((pool, nkv, bs, D), float("nan"), device="cuda", dtype=dtype)
    vc = torch.full_like(kc, float("nan"))
    pos = torch.arange(total, device="cuda")
    blk = bt[0].long()[pos // bs]
    kc[blk, :, pos % bs] = (torch.randn(total, nkv, D, device="cuda", generator=g) * 0.5).to(dtype)
    vc[blk, :, pos % bs] = (torch.randn(total, nkv, D, device="cuda", generator=g) * 0.5).to(dtype)
    return kc, vc, bt


@pytest.mark.parametrize("past,n", [(1, 2), (63, 5), (1000, 8), (6000, 16)])
def test_verify_row_equals_successive_decode(past, n):
    g = torch.Generator(device="cuda").manual_seed(past)
    nh, nkv, bs = 8, 2, 64
    kc, vc, bt = _cache(past, n, nkv, bs, torch.bfloat16, g)
    q = (torch.randn(n, nh, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    scale = 1.0 / math.sqrt(D)
    out = torch.zeros(n, nh * D, device="cuda", dtype=torch.bfloat16)
    _ext().decode_attention_paged_multi(q, kc, vc, bt, i32(0), i32(n), i32(past), scale, out)
    assert torch.isfinite(out.float()).all()
    for j in range(n):
        one = _ext().decode_attention_paged(q[j:j + 1].contiguous(), kc, vc, i32(past + j + 1), bt, scale)
        assert rel_err(out[j], one.reshape(-1)) < 2e-2, j


@pytest.mark.parametrize("kv", [torch.int8, torch.float8_e4m3fn])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quantized_multi_decode_is_bitwise_the_16bit_kernel(dtype, kv):
    """Three sequences of 2 / 5 / 8 new tokens over 1000 / 63 / 6000 cached ones: the 8-bit instantiations equal the 16-bit one on the
    dequantized cache."""
    g = torch.Generator(device="cuda").manual_seed(1)
    nh, nkv, bs = 8, 2, 16
    seqs = [(1000, 2), (63, 5), (6000, 8)]
    nblk = [(p + n + bs - 1) // bs for p, n in seqs]
    pool = sum(nblk) + 4
    perm = torch.randperm(pool, device="cuda", generator=g).to(torch.int32)
    bt = torch.full((len(seqs), max(nblk)), int(perm[-1]), dtype=torch.int32, device="cuda")
    o = 0
    for i, k in enumerate(nblk):
        bt[i, :k] = perm[o:o + k]
        o += k
    kc8, vc8 = _random_8bit((pool, nkv, bs, D), kv, g), _random_8bit((pool, nkv, bs, D), kv, g)
    kdq, vdq = _pow2_scales(nkv, 5), _pow2_scales(nkv, 6)
    kc16 = (kc8.float() * kdq[None, :, None, None]).to(dtype)
    vc16 = (vc8.float() * vdq[None, :, None, None]).to(dtype)
    t = sum(n for _, n in seqs)
    q = (torch.randn(t, nh, D, device="cuda", generator=g) * 0.5).to(dtype)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    cu, nq, past = i32([0, 2, 7]), i32([n for _, n in seqs]), i32([p for p, _ in seqs])
    scale = 1.0 / math.sqrt(D)
    outs = []
    for kc, vc, dq in ((kc8, vc8, dict(k_dequant_scales=kdq, v_dequant_scales=vdq)), (kc16, vc16, {})):
        out = torch.zeros(t, nh * D, device="cuda", dtype=dtype)
        _ext().decode_attention_paged_multi(q, kc, vc, bt, cu, nq, past, scale, out, **dq)
        outs.append(out)
    assert torch.isfinite(outs[0].float()).all()
    assert torch.equal(outs[0], outs[1])


def test_short_rows_never_call_the_prefill_kernel_or_the_reference(monkeypatch):
    specs = [(0, 7, 1), (0, 1000, 2), (0, 63, 5), (0, 64, min(PA.VERIFY_MAX, 16))]
    qkv, kc, vc, args = _batch(specs, 8, 2, 64, torch.bfloat16, seed=2)

    def boom(*a, **k):
        raise AssertionError("unexpected call on the short-row path")

    monkeypatch.setattr(PA, "_block_attention_ref", boom)
    monkeypatch.setattr(_ext(), "attention_fwd_paged", boom)
    out, _, _, _ = PA.block_attention(qkv, kc, vc, *args)
    assert torch.isfinite(out.as_subclass(torch.Tensor).float()).all()


def test_engine_verify_logits_match_plain_decode():
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.llama_tiny(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                                vocab_size=512, max_position_embeddings=1024)
        m = models.LlamaForCausalLM(cfg)
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    g = torch.Generator().manual_seed(0)
    prompt = torch.randint(1, cfg.vocab_size, (200,), generator=g).tolist()
    n = 16
    plain = models.LLMEngine(m, num_blocks=64, block_size=16)
    calls = []
    fwd = plain._forward
    plain._forward = lambda *a, _f=fwd, _c=calls: _c.append(_f(*a)) or _c[-1]
    plain.add_request(prompt, n)
    ref = plain.run_until_done()[0]
    spec = models.LLMEngine(m, num_blocks=64, block_size=16, draft_model=m, num_speculative_tokens=4)
    verifies = []
    run = spec._run

    def record(net, seqs, n_new, enc, dec, toks=None, rows=None):
        out = run(net, seqs, n_new, enc, dec, toks, rows)
        if net is spec._target and n_new[0] > 1 and enc[0] == 0:
            verifies.append((dec[0], toks[0], out))
        return out

    spec._run = record
    spec.add_request(prompt, n)
    out = spec.run_until_done()[0]
    assert len(out) == n and verifies
    checked = 0
    for c, toks, logits in verifies:
        done = c - len(prompt)                                     # generated tokens already in the cache
        if out[:done] != ref[:done]:                               # bf16 near-ties may send the two engines down different paths
            break
        for i in range(len(toks)):
            gen = done + 1 + i                                     # the generated index row i predicts
            if gen >= n or toks[:i + 1] != ref[done:gen]:          # past the end, or fed a token plain decoding did not see
                break
            assert rel_err(logits[i].float(), calls[gen][0].float()) < 2e-2, (c, i)
            checked += 1
    assert checked >= 2


def test_multi_decode_kernels_use_no_local_memory():
    obj = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddle_b200", "_build_cache", "decode_attention.cuda.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    multi = [f for f in funcs if "decode_multi" in f.split("\n", 1)[0]]
    assert len(multi) == 8                                        # split kernels (2 dtypes x 16-bit / int8 / fp8) and 2 merge kernels
    for f in multi:
        name = f.split("\n", 1)[0]
        assert not re.search(r"\b(LDL|STL)\b", f), name
        if "split_kernel" in name:
            assert re.search(r"\bHMMA\.16816\.F32", f), name         # tensor-core mma.sync; no wgmma, so no warpgroup fences to count
            assert "WARPGROUP" not in f, name
