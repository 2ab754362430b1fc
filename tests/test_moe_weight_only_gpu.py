"""Weight-only int8 / int4 MoE experts on the H100 (needs a GPU): the grouped in-SM expert GEMM (csrc/gemm_wo_sm100.cu) against an fp64
per-expert product of the dequantised weights, idle experts never read, the batched dequantisation bit for bit against the torch
expression, exact launch counts and no host synchronisation on the in-SM route, the dequantise route bit for bit against the 16-bit
grouped path, no local memory in the new kernels, and LLMEngine serving an int4-g128 expert-quantised Mixtral."""
import copy
import functools
import os
import re
import subprocess

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import _build, kernels, models
from paddle_b200.kernels import moe as KM
from paddle_b200.nn import quant as Q
from test_paged_prefill_gpu import rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(t):
    return t.as_subclass(paddle.Tensor)


@functools.lru_cache(maxsize=None)
def _stack(wdt, gs, E, k, n):
    """Stacked weight_quantize outputs q [E, n, k] (int4 [E, n, k/2]), fp32 scales and the fp64 dequantised stack [E, k, n]."""
    g = torch.Generator(device="cuda").manual_seed(E * 7 + k + n)
    w = torch.randn(E, k, n, device="cuda", generator=g) * 0.05
    w[:, : k // 2] *= 8.0                                            # scales that differ from group to group
    qs = [Q.weight_quantize(_p(w[e]), algo=f"weight_only_{wdt}", group_size=gs) for e in range(E)]
    q = torch.stack([q.as_subclass(torch.Tensor) for q, _ in qs]).contiguous()
    s = torch.stack([s.as_subclass(torch.Tensor).float() for _, s in qs]).contiguous()
    d = torch.stack([Q._dequantize_torch(q[e], s[e], wdt == "int4", torch.float64, gs) for e in range(E)])
    return q, s, d


def _routing(S, E, pattern, gen):
    if pattern == "spread":
        idx = torch.randint(0, E, (S,), device="cuda", generator=gen)
    elif pattern == "few":                                           # most experts idle
        idx = torch.tensor([1, 5, E - 1], device="cuda")[torch.randint(0, 3, (S,), device="cuda", generator=gen)]
    elif pattern == "one":                                           # one expert holds every slot
        idx = torch.full((S,), E // 2, device="cuda")
    else:                                                            # dropped slots
        idx = torch.randint(0, E, (S,), device="cuda", generator=gen)
        idx[torch.rand(S, device="cuda", generator=gen) < 0.3] = -1
    return idx.long()


# experts x routing pattern x activation dtype x bias: E = 64 leaves most experts idle
CASES = [(8, "spread", torch.bfloat16, True), (64, "few", torch.float16, False), (8, "one", torch.bfloat16, False),
         (8, "dropped", torch.float16, True)]


# k = 1408: 22 k-blocks (ragged int4 raw boxes); n = 1000: a partial channel tile; 5120 x 256: few channel tiles, cluster split-K
@pytest.mark.parametrize("wdt,gs", [("int8", -1), ("int8", 64), ("int8", 128), ("int4", -1), ("int4", 64), ("int4", 128)])
@pytest.mark.parametrize("k,n", [(1408, 1000), (5120, 256)])
@pytest.mark.parametrize("S", [1, 5, 16, 17, 64, 300])
@pytest.mark.parametrize("E,pattern,dtype,bias", CASES)
def test_expert_kernel_against_fp64(wdt, gs, k, n, S, E, pattern, dtype, bias):
    C = _build.ext()
    q, s, d = _stack(wdt, gs, E, k, n)
    gen = torch.Generator(device="cuda").manual_seed(S * 31 + E)
    idx = _routing(S, E, pattern, gen)
    x = (torch.randn(S, k, device="cuda", generator=gen) * 0.5).to(dtype)
    b = (torch.randn(E, n, device="cuda", generator=gen) * 0.1).to(dtype) if bias else None
    idle = torch.ones(E, dtype=torch.bool, device="cuda")
    idle[idx[idx >= 0]] = False
    s = s.clone()
    s[idle] = float("nan")                                           # experts nobody selected: their scales and bias are never read
    if b is not None:
        b[idle] = float("nan")
    kernels.reset_launch_count()
    dest, offsets, work = C.moe_wo_plan(idx, E)
    xp = C.moe_rows_scatter(x, dest, None, 1, S)
    y = C.weight_only_gemm_experts(xp, q, s, b, offsets, work, wdt == "int4", gs)
    assert kernels.launch_count() == 3 + 1 + 1
    assert y.shape == (S, n) and y.dtype == dtype
    live = idx >= 0
    got = y[dest[live].long()]
    assert bool(torch.isfinite(got).all())
    ref = torch.empty(got.shape, dtype=torch.float64, device="cuda")
    for e in idx[live].unique().tolist():                             # slot i of expert e: x[i] @ dequant(W[e]) + b[e]
        sel = idx[live] == e
        ref[sel] = x[live][sel].double() @ d[e] + (0 if b is None else b[e].double())
    assert rel_err(got, ref) < 1e-2, rel_err(got, ref)
    off = offsets.tolist()
    assert off[0] == 0 and off[-1] == int(live.sum()) and all(a <= c for a, c in zip(off, off[1:]))


@pytest.mark.parametrize("wdt", ["int8", "int4"])
@pytest.mark.parametrize("gs", [-1, 64, 128])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_batched_dequantize_equals_the_torch_expression(wdt, gs, out_dtype):
    q, s, _ = _stack(wdt, gs, 8, 1408, 1000)
    kernels.reset_launch_count()
    got = KM.dequantize_experts(q, s, wdt == "int4", gs, out_dtype)
    assert kernels.launch_count() == 1
    assert got.shape == (8, 1408, 1000) and got.dtype == out_dtype and got.is_contiguous()
    for e in range(8):
        ref = Q._dequantize_torch(q[e], s[e], wdt == "int4", out_dtype, gs)
        assert torch.equal(got[e].view(torch.int16 if out_dtype != torch.float32 else torch.int32),
                           ref.view(torch.int16 if out_dtype != torch.float32 else torch.int32)), e


def _ffn_inputs(T, topk, E, d, f, wdt, gs, dtype=torch.bfloat16, seed=0):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(T, d, device="cuda", generator=gen) * 0.5).to(dtype)
    logits = torch.randn(T, E, device="cuda", generator=gen)
    val, idx = torch.softmax(logits, -1).topk(topk, -1)
    q1, s1, _ = _stack(wdt, gs, E, d, 2 * f)
    q2, s2, _ = _stack(wdt, gs, E, f, d)
    return x, idx, (val / val.sum(-1, keepdim=True)).float(), q1, s1, q2, s2


def test_in_sm_route_launches_and_never_syncs():
    T, topk = KM.WO_MOE_MAX_SLOTS // 2, 2
    x, idx, w, q1, s1, q2, s2 = _ffn_inputs(T, topk, 8, 512, 1024, "int4", 128)
    KM.expert_ffn_weight_only(x, idx, w, q1, s1, q2, s2, True, 128)     # warm-up: module loads and tensor maps
    torch.cuda.synchronize()
    kernels.reset_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = KM.expert_ffn_weight_only(x, idx, w, q1, s1, q2, s2, True, 128)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    # plan (count, plan, dest) + scatter + GEMM 1 + SwiGLU + GEMM 2 + combine
    assert kernels.launch_count() == 3 + 1 + 1 + 1 + 1 + 1
    C = _build.ext()
    C.tracer_collect()
    C.tracer_enable(1)
    try:
        y2 = KM.expert_ffn_weight_only(x, idx, w, q1, s1, q2, s2, True, 128)
        torch.cuda.synchronize()
    finally:
        C.tracer_enable(0)
    names = [e[0] for e in C.tracer_collect()]
    assert torch.equal(y, y2)
    assert names.count("weight_only_gemm_experts") == 2 and not any("dequantize" in nm for nm in names)
    # against the dequantise route on the same weights
    ref = KM.expert_ffn_grouped(x, idx, w, KM.dequantize_experts(q1, s1, True, 128, x.dtype), KM.dequantize_experts(q2, s2, True, 128, x.dtype))
    assert rel_err(y, ref) < 2e-2


@pytest.mark.parametrize("wdt,gs", [("int8", -1), ("int4", 128)])
def test_dequantize_route_is_bitwise_the_16bit_grouped_path(wdt, gs):
    T, topk = KM.WO_MOE_MAX_SLOTS // 2 + 1, 2                         # one slot pair past the in-SM route
    x, idx, w, q1, s1, q2, s2 = _ffn_inputs(T, topk, 8, 512, 1024, wdt, gs, seed=1)
    int4 = wdt == "int4"
    kernels.reset_launch_count()
    y = KM.expert_ffn_weight_only(x, idx, w, q1, s1, q2, s2, int4, gs)
    # dequantise ffn1 + route (count, plan, dest) + scatter + grouped GEMM + SwiGLU + dequantise ffn2 + grouped GEMM + combine
    assert kernels.launch_count() == 1 + 3 + 1 + 1 + 1 + 1 + 1 + 1
    w1 = KM.dequantize_experts(q1, s1, int4, gs, x.dtype)
    w2 = KM.dequantize_experts(q2, s2, int4, gs, x.dtype)
    assert torch.equal(y, KM.expert_ffn_grouped(x, idx, w, w1, w2))


def test_fused_moe_quantized_on_the_gpu():
    from paddle_b200.incubate.nn import functional as IF

    gen = torch.Generator(device="cuda").manual_seed(5)
    E, d, f = 8, 512, 1024
    x = (torch.randn(3, d, device="cuda", generator=gen)).to(torch.bfloat16)
    gate = torch.randn(d, E, device="cuda", generator=gen)
    q1, s1, d1 = _stack("int8", 64, E, d, 2 * f)
    q2, s2, d2 = _stack("int8", 64, E, f, d)
    b1 = (torch.randn(E, 1, 2 * f, device="cuda", generator=gen) * 0.1).to(torch.bfloat16)
    b2 = (torch.randn(E, 1, d, device="cuda", generator=gen) * 0.1).to(torch.bfloat16)
    kernels.reset_launch_count()
    out = IF.fused_moe(_p(x), _p(gate), _p(q1), _p(q2), _p(b1), _p(s1), _p(b2), _p(s2), quant_method="weight_only_int8").as_subclass(torch.Tensor)
    assert kernels.launch_count() == 8                                # 6 slots: the in-SM route, biases in the GEMM epilogues
    val, idx = torch.softmax(x.float() @ gate, -1).topk(2, -1)       # the routing of fused_moe, then fp64 experts
    val = (val / val.sum(-1, keepdim=True)).double()
    ref = torch.zeros(3, d, dtype=torch.float64, device="cuda")
    for t in range(3):
        for j in range(2):
            e = int(idx[t, j])
            h = x[t].double() @ d1[e] + b1[e, 0].double()
            a = torch.nn.functional.silu(h[:f]) * h[f:]
            ref[t] += val[t, j] * (a @ d2[e] + b2[e, 0].double())
    assert rel_err(out, ref) < 2e-2


def test_expert_gemm_plan_and_dequant_kernels_use_no_local_memory():
    found = 0
    for obj in ("gemm_wo_sm100.cuda.o", "moe.cuda.o"):
        sass = subprocess.run(["cuobjdump", "-sass", os.path.join(ROOT, "paddle_b200", "_build_cache", obj)], capture_output=True, text=True,
                              check=True).stdout
        for f in re.split(r"\n\s*Function : ", sass)[1:]:
            name, body = f.split("\n", 1)
            # the expert GEMM: wo_gemm_kernel's instantiations with EXPERTS = true, its last template argument
            if re.search(r"wo_gemm_kernelI(?:L[ib]\d+E){5}Lb1E", name) or "moe_wo_plan_kernel" in name or "wo_dequant_kernel" in name:
                found += 1
                assert not re.search(r"\b(LDL|STL)\b", body), name
    assert found == 2 * 2 * 2 * 3 + 1 + 2 * 3                          # tile x int8 / int4 x bf16 / fp16 x group; plan; dequantisation


def _mixtral_pair():
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.mixtral_tiny(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                                  num_local_experts=8, vocab_size=512, max_position_embeddings=1024)
        ref = models.MixtralForCausalLM(cfg)
        ref.eval()
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    qm = models.quantize_weights(copy.deepcopy(ref), "weight_only_int4", 128, experts=True)
    from paddle_b200.models.weight_only import _targets

    d = copy.deepcopy(ref)                                           # the 16-bit model holding the dequantised weights
    with torch.no_grad():
        for (qp, name), (dp, _) in zip(_targets(qm), _targets(d)):
            getattr(dp, name).weight.as_subclass(torch.Tensor).copy_(getattr(qp, name).dequantized_weight(torch.bfloat16).as_subclass(torch.Tensor))
        for ql, dl in zip(qm.layers, d.layers):
            w1, w2 = ql.moe.experts.dequantized(torch.bfloat16)
            dl.moe.experts.w1.as_subclass(torch.Tensor).copy_(w1)
            dl.moe.experts.w2.as_subclass(torch.Tensor).copy_(w2)
    return qm, d, cfg


def test_engine_int4_g128_expert_quantized_mixtral_against_the_dequantized_model():
    qm, d, cfg = _mixtral_pair()
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in (900, 700, 800)]   # prefill: past WO_MOE_MAX_SLOTS
    n = 8
    C = _build.ext()

    def serve(model, trace):
        eng = models.LLMEngine(model, num_blocks=256, block_size=16)
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
    assert rows * cfg.num_experts_per_tok > KM.WO_MOE_MAX_SLOTS and steps_d[0][0] == rows
    assert "weight_dequantize_experts" in names and "weight_only_gemm_experts" not in names
    for key, v in logits_q.items():                                  # dequantise + the 16-bit grouped GEMM: the same bits
        assert torch.equal(v, steps_d[0][1][key]), key
    decode = [(r, lg, nm) for r, lg, nm in steps_q[1:] if r * cfg.num_experts_per_tok <= KM.WO_MOE_MAX_SLOTS]
    assert decode
    ref_logits = {k: v for _, lg, _ in steps_d[1:] for k, v in lg.items()}
    checked = 0
    for r, lg, nm in decode:
        assert "weight_only_gemm_experts" in nm and not any("dequantize" in x for x in nm)   # the in-SM kernel, no dequantisation
        for (sid, pos), v in lg.items():
            j = pos - len(prompts[sid])
            if out_q[sid][:j] != out_d[sid][:j]:
                continue                                             # the two models already chose different tokens
            assert rel_err(v, ref_logits[(sid, pos)]) < 2e-2, (sid, pos)
            checked += 1
    assert checked >= 6
