"""Group-wise weight-only GEMM (csrc/gemm_wo_sm100.cu, group_size 64 / 128) against an fp64 product of the dequantised weight, the
one-pass dequantisation kernel bit for bit against the torch expression, the bindings' operand checks, and LLMEngine serving an
int4-g128 Llama: decode steps on the in-SM kernel, larger steps on dequantise + GEMM (needs a GPU)."""
import copy

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import _build, kernels, models
from paddle_b200.nn import quant as Q
from test_paged_prefill_gpu import rel_err

pytestmark = pytest.mark.gpu

# k = 1408: 22 k-blocks (ragged int4 raw boxes, uneven split ranks); 5120: many ring phases; 11008 x 256: few channel tiles, cluster split-K.
# n = 1000: a partial channel tile.
SHAPES = [(1408, 1000), (1408, 1536), (5120, 1000), (5120, 1536), (11008, 256)]


def _p(t):
    return t.as_subclass(paddle.Tensor)


@pytest.mark.parametrize("wdt,gs", [("int8", 64), ("int8", 128), ("int4", 64), ("int4", 128)])
@pytest.mark.parametrize("k,n", SHAPES)
@pytest.mark.parametrize("m", [1, 5, 16, 17, 48, 64])
@pytest.mark.parametrize("dtype,bias", [(torch.bfloat16, True), (torch.float16, False), (torch.bfloat16, False), (torch.float16, True)])
def test_grouped_kernel_against_fp64(wdt, gs, k, n, m, dtype, bias):
    g = torch.Generator(device="cuda").manual_seed(k + n + m)
    w = torch.randn(k, n, device="cuda", generator=g) * 0.05
    w[: k // 2] *= 8.0                                               # scales that differ from group to group
    x = (torch.randn(m, k, device="cuda", generator=g) * 0.5).to(dtype)
    b = (torch.randn(n, device="cuda", generator=g) * 0.1).to(dtype) if bias else None
    wq, sc = Q.weight_quantize(_p(w), algo=f"weight_only_{wdt}", group_size=gs)
    kernels.reset_launch_count()
    y = Q.weight_only_linear(_p(x), wq, None if b is None else _p(b), sc, wdt, group_size=gs).as_subclass(torch.Tensor)
    assert kernels.launch_count() == 1
    assert y.shape == (m, n) and y.dtype == dtype
    wd = Q._dequantize_torch(wq.as_subclass(torch.Tensor), sc.as_subclass(torch.Tensor), wdt == "int4", torch.float64, gs)
    ref = x.double() @ wd + (0 if b is None else b.double())
    assert rel_err(y, ref) < 1e-2, rel_err(y, ref)


@pytest.mark.parametrize("wdt", ["int8", "int4"])
@pytest.mark.parametrize("gs", [-1, 64, 128])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("k,n", [(1408, 1000), (256, 77), (5120, 13824)])
def test_dequantize_kernel_equals_the_torch_expression(wdt, gs, out_dtype, k, n):
    if gs == -1 and wdt == "int8":
        k += 2                                                       # per-channel: any even fan-in
    g = torch.Generator(device="cuda").manual_seed(k * n)
    w = torch.randn(k, n, device="cuda", generator=g)
    wq, sc = Q.weight_quantize(_p(w), algo=f"weight_only_{wdt}", group_size=gs)
    kernels.reset_launch_count()
    got = Q.weight_dequantize(wq, sc, f"weight_only_{wdt}", out_dtype, gs).as_subclass(torch.Tensor)
    assert kernels.launch_count() == 1
    ref = Q._dequantize_torch(wq.as_subclass(torch.Tensor), sc.as_subclass(torch.Tensor), wdt == "int4", out_dtype, gs)
    assert got.shape == (k, n) and got.dtype == out_dtype and got.is_contiguous()
    assert torch.equal(got.view(torch.int16 if out_dtype != torch.float32 else torch.int32),
                       ref.view(torch.int16 if out_dtype != torch.float32 else torch.int32))
    # 16-bit scales go through fp32 exactly as the torch path does
    sc16 = sc.as_subclass(torch.Tensor).to(torch.bfloat16)
    got16 = Q.weight_dequantize(wq, _p(sc16), f"weight_only_{wdt}", out_dtype, gs).as_subclass(torch.Tensor)
    assert torch.equal(got16, Q._dequantize_torch(wq.as_subclass(torch.Tensor), sc16, wdt == "int4", out_dtype, gs))


def test_binding_checks_the_scale_for_each_mode():
    C = _build.ext()
    x = torch.randn(4, 256, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(64, 256, device="cuda", dtype=torch.int8)
    with pytest.raises(RuntimeError, match=r"scale float32 \[K / group_size, N\]"):
        C.weight_only_gemm(x, w, torch.ones(64, device="cuda"), None, False, 64)
    with pytest.raises(RuntimeError, match=r"scale float32 \[N\]"):
        C.weight_only_gemm(x, w, torch.ones(4, 64, device="cuda"), None, False, -1)
    with pytest.raises(RuntimeError, match="group_size"):
        C.weight_only_gemm(x, w, torch.ones(8, 64, device="cuda"), None, False, 32)
    with pytest.raises(RuntimeError, match="contiguous"):
        C.weight_only_gemm(x, w, torch.ones(64, 4, device="cuda").t(), None, False, 64)
    with pytest.raises(RuntimeError, match="multiple of group_size"):
        C.weight_dequantize(w[:, :192].contiguous(), torch.ones(1, 64, device="cuda"), False, 128, torch.bfloat16)


def _expert_operands(dev):
    """A 2-expert weight_only_gemm_experts call on `dev`: xp, w, scale, bias, offsets, work (the plan of 4 routed rows)."""
    C = _build.ext()
    _, offsets, work = C.moe_wo_plan(torch.tensor([0, 1, 1, 0], device=dev), 2)
    return (torch.randn(4, 256, device=dev, dtype=torch.bfloat16), torch.zeros(2, 64, 256, device=dev, dtype=torch.int8),
            torch.ones(2, 64, device=dev), torch.zeros(2, 64, device=dev, dtype=torch.bfloat16), offsets, work)


def test_bindings_reject_a_cpu_bias():
    C = _build.ext()
    x = torch.randn(4, 256, device="cuda", dtype=torch.bfloat16)
    w = torch.zeros(64, 256, device="cuda", dtype=torch.int8)
    with pytest.raises(RuntimeError, match="bias"):
        C.weight_only_gemm(x, w, torch.ones(64, device="cuda"), torch.zeros(64, dtype=torch.bfloat16), False, -1)
    xp, w3, s3, b3, offsets, work = _expert_operands("cuda")
    with pytest.raises(RuntimeError, match="bias"):
        C.weight_only_gemm_experts(xp, w3, s3, b3.cpu(), offsets, work, False, -1)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_bindings_reject_operands_on_another_device():
    C = _build.ext()
    x = torch.randn(4, 256, device="cuda:0", dtype=torch.bfloat16)
    w = torch.zeros(64, 256, device="cuda:0", dtype=torch.int8)
    sc, b = torch.ones(64, device="cuda:0"), torch.zeros(64, device="cuda:0", dtype=torch.bfloat16)
    for args in ((w, sc, b.to("cuda:1")), (w, sc.to("cuda:1"), b), (w.to("cuda:1"), sc.to("cuda:1"), b)):
        with pytest.raises(RuntimeError, match="one device"):
            C.weight_only_gemm(x, *args, False, -1)
    xp, w3, s3, b3, offsets, work = _expert_operands("cuda:0")
    for args in ((w3, s3, b3.to("cuda:1")), (w3, s3.to("cuda:1"), b3)):
        with pytest.raises(RuntimeError, match="one device"):
            C.weight_only_gemm_experts(xp, *args, offsets, work, False, -1)


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
    qm = models.quantize_weights(copy.deepcopy(ref), "weight_only_int4", 128)
    from paddle_b200.models.weight_only import _targets

    d = copy.deepcopy(ref)                                           # the 16-bit model holding the dequantised weights
    for (qp, name), (dp, _) in zip(_targets(qm), _targets(d)):
        with torch.no_grad():
            getattr(dp, name).weight.as_subclass(torch.Tensor).copy_(getattr(qp, name).dequantized_weight(torch.bfloat16).as_subclass(torch.Tensor))
    return qm, d, cfg


def test_engine_int4_g128_llama_against_the_dequantized_model():
    qm, d, cfg = _llama_pair()
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in (90, 70, 130)]
    n = 8
    C = _build.ext()

    def serve(model, trace):
        eng = models.LLMEngine(model, num_blocks=128, block_size=16)
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
    rows, logits_q, names = steps_q[0]
    assert rows > 64 and steps_d[0][0] == rows
    assert "weight_dequantize" in names and "weight_only_gemm" not in names
    for key, v in logits_q.items():                                  # dequantise + the 16-bit GEMM: the same bits
        assert torch.equal(v, steps_d[0][1][key]), key
    decode = [(r, lg, nm) for r, lg, nm in steps_q[1:] if r <= 64]
    assert decode
    ref_logits = {k: v for _, lg, _ in steps_d[1:] for k, v in lg.items()}
    checked = 0
    for r, lg, nm in decode:
        assert "weight_only_gemm" in nm and "weight_dequantize" not in nm      # the in-SM kernel, no dequantisation
        for (sid, pos), v in lg.items():
            j = pos - len(prompts[sid])
            if out_q[sid][:j] != out_d[sid][:j]:
                continue                                             # the two models already chose different tokens
            assert rel_err(v, ref_logits[(sid, pos)]) < 2e-2, (sid, pos)
            checked += 1
    assert checked >= 6
