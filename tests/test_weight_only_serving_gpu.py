"""Group-wise weight-only GEMM (csrc/gemm_wo_sm100.cu, group_size 64 / 128) against an fp64 product of the dequantised weight, the
one-pass dequantisation kernel bit for bit against the torch expression, the per-channel instantiations' unchanged SASS, and LLMEngine
serving an int4-g128 Llama: decode steps on the in-SM kernel, larger steps on dequantise + GEMM (needs a GPU)."""
import copy
import hashlib
import json
import os
import re
import subprocess

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import _build, kernels, models
from paddle_b200.nn import quant as Q
from test_paged_prefill_gpu import rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
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


def _sass_functions():
    obj = os.path.join(ROOT, "paddle_b200", "_build_cache", "gemm_wo_sm100.cuda.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = f.split("\n", 1)
        out[name.strip()] = [re.sub(r"/\*[0-9a-f]{4}\*/", "", ln).strip() for ln in body.split("\n") if re.search(r"/\*[0-9a-f]{4}\*/", ln)]
    return out


def test_wo_kernels_sass():
    funcs = _sass_functions()
    per_channel, grouped = {}, []
    for name, ins in funcs.items():
        mt = re.search(r"wo_gemm_kernelI((?:L[ib]\d+E)+)E", name)
        if mt is None:
            continue
        ntok, wst, int4, bf16, gs = (int(v) for v in re.findall(r"L[ib](\d+)E", mt.group(1)))
        if gs == 0:
            per_channel[f"NTOK={ntok},WST={wst},INT4={int4},BF16={bf16}"] = hashlib.sha256("\n".join(ins).encode()).hexdigest()
        else:
            grouped.append(name)
    assert len(grouped) == 2 * 2 * 2 * 2                             # token tile x int8 / int4 x bf16 / fp16 x group 64 / 128
    for name, ins in funcs.items():
        if "wo_gemm_kernel" in name or "wo_dequant_kernel" in name:
            assert not any(re.search(r"\b(LDL|STL)\b", i) for i in ins), name
    # the per-channel instantiations compile to the instructions they compiled to before group-wise scales were added
    with open(os.path.join(ROOT, "tests", "golden", "wo_gemm_per_channel_sass.json")) as f:
        assert per_channel == json.load(f)


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
