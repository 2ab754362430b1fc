"""int8 activations on the H100: the int8 wgmma GEMM (int32 and dequantising epilogues), the per-token quantizer, llm_int8_linear and an
llm.int8 model served by LLMEngine, against int64 / float64 evaluations and the torch expressions they reproduce."""
import copy
import os
import re
import subprocess

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import _build, kernels, models
from paddle_b200.kernels import gemm_int8 as G8
from paddle_b200.nn import quant as Q
from test_paged_prefill_gpu import rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(t):
    return t.as_subclass(paddle.Tensor)


def _r(t):
    return t.as_subclass(torch.Tensor)


def _operand(rows, k, g):
    """int8 [rows, k] on the GPU: random values, with -128 / -127 / 127 planted everywhere (the largest products)."""
    t = torch.randint(-128, 128, (rows, k), generator=g, dtype=torch.int8)
    pick = torch.rand(rows, k, generator=g)
    t[pick < 0.15] = -128
    t[(pick >= 0.15) & (pick < 0.25)] = 127
    t[(pick >= 0.25) & (pick < 0.3)] = -127
    return t.cuda()


def _exact(a, b):
    """a @ b^T as int64 (the float64 product of int8 operands is exact here: |sum| <= 11008 * 2^14 < 2^53)."""
    return (a.double() @ b.double().transpose(-1, -2)).long()


@pytest.mark.parametrize("k", [16, 48, 1040, 4096, 11008])
@pytest.mark.parametrize("n", [8, 1000, 4096, 12288])
def test_int32_epilogue_is_exact(k, n):
    g = torch.Generator().manual_seed(k * 7 + n)
    b = _operand(n, k, g)
    for m in (1, 7, 64, 128, 129, 1000, 4096):
        a = _operand(m, k, g)
        out = _r(paddle.matmul(_p(a), _p(b), transpose_y=True))
        assert out.dtype == torch.int32 and out.shape == (m, n)
        assert torch.equal(out.long(), _exact(a, b)), (m, n, k)
    worst = torch.full((129, k), -128, dtype=torch.int8, device="cuda")
    assert (_r(paddle.matmul(_p(worst), _p(worst), transpose_y=True)) == k * 128 * 128).all()


def test_int32_batched_transpose_and_fallbacks():
    g = torch.Generator().manual_seed(5)
    a = torch.stack([_operand(200, 1040, g) for _ in range(3)])
    b = torch.stack([_operand(300, 1040, g) for _ in range(3)])
    ref = _exact(a, b)
    kernels.reset_launch_count()
    out = _r(paddle.matmul(_p(a), _p(b), transpose_y=True))
    assert kernels.launch_count() == 1 and out.dtype == torch.int32 and torch.equal(out.long(), ref)
    bt = b.transpose(1, 2).contiguous()                                  # [B, K, N]: transpose_y=False
    assert torch.equal(_r(paddle.matmul(_p(a), _p(bt))).long(), ref)
    at = a.transpose(1, 2).contiguous()
    assert torch.equal(_r(paddle.matmul(_p(at), _p(bt), transpose_x=True)).long(), ref)
    assert torch.equal(_r(paddle.matmul(_p(a[0]), _p(bt[0]))).long(), ref[0])
    odd_a, odd_b = _operand(33, 40, g), _operand(20, 40, g)             # K % 16 != 0: the exact fallback
    assert torch.equal(_r(paddle.matmul(_p(odd_a), _p(odd_b), transpose_y=True)).long(), _exact(odd_a, odd_b))
    out = _r(paddle.matmul(_p(a), _p(bt[:1])))                           # broadcasting batch
    assert out.dtype == torch.int32 and torch.equal(out.long(), _exact(a, b[:1].expand(3, -1, -1)))


def _activations(m, k, dtype, g):
    x = (torch.randn(m, k, generator=g) * 2).to(dtype)
    x[3] = 0                                                             # all-zero row
    x[5] = 0
    x[5, 0], x[5, 1], x[5, 2], x[5, 3] = 127.0, 2.5, -3.5, 0.5           # row scale 1: quotients land exactly on .5
    x[6, :8] = torch.tensor([1e-3, -7e-4, 2e-3, 0, 0, 0, 0, 0]).to(dtype)
    x[6, 8:] = 0                                                         # tiny row
    return x.cuda()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("m,k", [(9, 16), (130, 4096), (1000, 11008)])
def test_quantizer_equals_the_torch_expression(dtype, m, k):
    g = torch.Generator().manual_seed(m + k)
    x = _activations(m, k, dtype, g)
    mask = torch.rand(k, generator=g) < 0.05
    for msk in (None, mask.cuda()):
        kernels.reset_launch_count()
        q, s = G8.quantize_int8_rows(x, msk)
        assert kernels.launch_count() == 1
        q_ref, s_ref = G8.quantize_int8_rows(x.cpu(), None if msk is None else msk.cpu())
        assert torch.equal(s.cpu(), s_ref) and torch.equal(q.cpu(), q_ref)
    assert q[5, :4].tolist() == [127, 2, -4, 0] and (q[3] == 0).all()


@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("m,n,k", [(7, 1000, 48), (300, 4096, 4096), (1000, 12288, 1040)])
def test_dequant_epilogue_equals_the_torch_expression(out_dtype, m, n, k):
    g = torch.Generator().manual_seed(m * n + k)
    a, b = _operand(m, k, g), _operand(n, k, g)
    rs = (torch.rand(m, generator=g) * 1e-2).cuda()
    cs = (torch.rand(n, generator=g) * 1e-3).cuda()
    bias = torch.randn(n, generator=g).cuda()
    for bb in (None, bias):
        y = G8.gemm_int8_dequant(a, b, rs, cs, bb, out_dtype)
        ref = G8.gemm_int8_dequant(a.cpu(), b.cpu(), rs.cpu(), cs.cpu(), None if bb is None else bb.cpu(), out_dtype)
        assert y.dtype == out_dtype and torch.equal(y.cpu(), ref), (bb is None)


def _linear_case(m, k, n, dtype, g, outliers=()):
    x = (torch.randn(m, k, generator=g)).to(dtype)
    for c in outliers:
        x[:, c] *= 30
    w = torch.randn(k, n, generator=g) * 0.02
    q, s = Q.weight_quantize(_p(w), algo="llm.int8")
    bias = (torch.randn(n, generator=g) * 0.1).to(dtype)
    return x.cuda(), _r(q).cuda(), _r(s).cuda(), bias.cuda()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_llm_int8_linear_threshold_inf_is_the_torch_path_in_two_launches(dtype):
    g = torch.Generator().manual_seed(11)
    x, q, s, bias = _linear_case(300, 4096, 1000, dtype, g)
    for b in (None, bias):
        kernels.reset_launch_count()
        y = _r(Q.llm_int8_linear(_p(x), _p(q), None if b is None else _p(b), _p(s), threshold=float("inf")))
        assert kernels.launch_count() == 2
        ref = _r(Q.llm_int8_linear(_p(x.cpu()), _p(q.cpu()), None if b is None else _p(b.cpu()), _p(s.cpu()), threshold=float("inf")))
        assert y.dtype == dtype and torch.equal(y.cpu(), ref)
    # row independence: every row equals, bit for bit, the same row computed alone
    y = _r(Q.llm_int8_linear(_p(x), _p(q), _p(bias), _p(s), threshold=float("inf")))
    for i in (0, 1, 63, 64, 127, 128, 299):
        yi = _r(Q.llm_int8_linear(_p(x[i:i + 1]), _p(q), _p(bias), _p(s), threshold=float("inf")))
        assert torch.equal(yi[0], y[i]), i


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_llm_int8_linear_with_outliers_against_float64(dtype):
    g = torch.Generator().manual_seed(12)
    k, n = 4096, 1000
    x, q, s, bias = _linear_case(257, k, n, dtype, g, outliers=(5, 900, 3001))
    y = _r(Q.llm_int8_linear(_p(x), _p(q), _p(bias), _p(s), threshold=6.0))
    x2 = x.double()
    out = (x2.abs() > 6.0).any(0)
    assert out.sum().item() >= 3
    xi = x2.masked_fill(out, 0.0)
    sx = xi.abs().amax(-1, keepdim=True).clamp(min=1e-8) / 127.0
    xq = torch.round(xi / sx).clamp(-128, 127)
    wd = _r(Q.weight_dequantize(_p(q), _p(s), "weight_only_int8", dtype)).double()
    ref = (xq @ q.double().t()) * sx * s.double() + x2[:, out] @ wd[out] + bias.double()
    assert rel_err(y.double(), ref) < 1e-2


def _llama_pair():
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.llama_tiny(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                                vocab_size=512, max_position_embeddings=1024)
        ref = models.LlamaForCausalLM(cfg)
        ref.eval()
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    qm = models.quantize_weights(copy.deepcopy(ref), "llm.int8", threshold=float("inf"))
    from paddle_b200.models.weight_only import _targets

    d = copy.deepcopy(ref)                                               # the 16-bit model holding the dequantised weights
    for (qp, name), (dp, _) in zip(_targets(qm), _targets(d)):
        with torch.no_grad():
            _r(getattr(dp, name).weight).copy_(_r(getattr(qp, name).dequantized_weight(torch.bfloat16)))
    return qm, d, cfg


def test_engine_llm_int8_llama_against_the_dequantized_model():
    qm, d, cfg = _llama_pair()
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in (90, 70, 130)]
    n = 8
    C = _build.ext()

    def serve(model, trace, **kw):
        eng = models.LLMEngine(model, num_blocks=128, block_size=16, **kw)
        steps = []
        fwd = eng._forward

        def record(seqs, n_new, enc, dec):
            if trace:
                C.tracer_collect()
                C.tracer_enable(1)
            try:
                out = fwd(seqs, n_new, enc, dec)
                torch.cuda.synchronize()
            finally:
                if trace:
                    C.tracer_enable(0)
            names = {e[0] for e in C.tracer_collect()} if trace else set()
            steps.append((sum(n_new), {(s.id, s.cached + k): out[i].float() for i, (s, k) in enumerate(zip(seqs, n_new))}, names))
            return out

        eng._forward = record
        ids = [eng.add_request(p, n) for p in prompts]
        res = eng.run_until_done()
        return [res[i] for i in ids], steps

    out_q, steps_q = serve(qm, True)
    out_d, steps_d = serve(d, False)
    assert steps_q[0][0] > 64
    for _, _, names in steps_q:
        assert {"gemm_int8_dequant", "quantize_int8_rows"} <= names
        assert "weight_dequantize" not in names and "weight_only_gemm" not in names
    ref_logits = {k: v for _, lg, _ in steps_d for k, v in lg.items()}
    checked = 0
    for _, lg, _ in steps_q:
        for (sid, pos), v in lg.items():
            j = pos - len(prompts[sid])                                  # the input token at pos is generated token j
            if j >= 0 and out_q[sid][:j + 1] != out_d[sid][:j + 1]:
                continue                                                 # the two models already chose different tokens
            # per-token int8 rounding of the activations: each of the four GEMM kinds adds 1-2 % to the logits of this random-weight
            # model (down_proj, whose SiLU * up inputs are heavy-tailed, the most); together 2.0-3.2 % was measured on an H100
            assert rel_err(v, ref_logits[(sid, pos)]) < 4e-2, (sid, pos)
            checked += 1
    assert checked >= 6
    out_c, _ = serve(qm, False, max_prefill_chunk=48)                    # chunked prefill: the same tokens
    assert out_c == out_q


def test_int8_gemm_sass():
    obj = os.path.join(ROOT, "paddle_b200", "_build_cache", "gemm_fp8_sm100.cuda.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = f.split("\n", 1)
        funcs[name.strip()] = body
    s8 = {k: v for k, v in funcs.items() if "gemm_s8_kernel" in k}
    assert len(s8) == 2                                                  # BN = 128, 256
    for name, body in s8.items():
        assert "IGMMA" in body, name
        assert not re.search(r"\b(LDL|STL)\b", body), name
        assert body.count("WARPGROUP.ARRIVE") < len(re.findall(r"\bIGMMA\.", body)), name
