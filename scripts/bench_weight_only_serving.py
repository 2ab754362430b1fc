"""Weight-only serving on the GPU: the in-SM dequantising GEMM (per-channel, group 64, group 128; int8 and int4) against the bf16 GEMM, the
one-pass dequantisation kernel against the torch expression, the two routes of weight_only_linear around its M <= 64 threshold, and
LLMEngine decode steps of a Llama-2-7B-shaped model with bf16, int8 per-channel and int4-g128 weights.

  kernel     Llama-2-7B and 13B projection shapes, m = 1 / 16 / 64 bf16 rows.  Each arm rotates through enough weight sets that they
             exceed the H100's 50 MB L2, so every call reads its weights from HBM.  Calls are captured into one CUDA graph (20 calls) and
             replayed; the median of 5 replays is reported per call.  GB/s counts the weight and scale bytes; "of_peak" divides by the
             data sheet's 3.35 TB/s.  The bf16 arm is `kernels.gemm.linear` (the project's wgmma GEMM; torch.matmul where it declines).
  dequant    13B gate_up (5120 x 27648): the CUDA kernel against the torch expression, median CUDA-event time of 10 runs, and the peak
             memory each allocates on top of its inputs.
  crossover  m = 64 / 128 / 256 rows through both routes: the in-SM kernel (64-row chunks above 64) and dequantise + GEMM.
  engine     decode-only steps of a random-weight Llama-2-7B-shaped model (32 layers) with 1 / 16 / 64 running sequences of 128-token
             prompts; each step is timed on the host between device synchronizes, --steps steps per round, --rounds rounds; the median
             and the spread (min, max) of the round medians are reported.

The card's name and power limit are read in the same run and printed with the numbers.

  python scripts/bench_weight_only_serving.py [--parts kernel,dequant,crossover,engine] [--steps N] [--rounds N] [--json FILE]
"""
import argparse
import copy
import json
import math
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_paged_prefill import gpu_identity  # noqa: E402
import paddle_b200 as paddle  # noqa: E402
from paddle_b200._build import ext  # noqa: E402
from paddle_b200.kernels import gemm as KG  # noqa: E402
from paddle_b200.nn import quant as Q  # noqa: E402

HBM = 3.35e12
L2 = 50 * 2 ** 20
SHAPES = {"7b": [("qkv", 4096, 12288), ("o", 4096, 4096), ("gate_up", 4096, 22016), ("down", 11008, 4096)],
          "13b": [("qkv", 5120, 15360), ("o", 5120, 5120), ("gate_up", 5120, 27648), ("down", 13824, 5120)]}
VARIANTS = [("int8", -1), ("int8", 64), ("int8", 128), ("int4", -1), ("int4", 64), ("int4", 128)]


def graph_time(fn, calls=20, replays=5):
    """Device time per call: `calls` calls captured into one CUDA graph, replayed; median replay over `replays`."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fn()
        st.synchronize()
        with torch.cuda.graph(g, stream=st):
            for _ in range(calls):
                fn()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    ts = []
    for _ in range(replays):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / calls)
    return statistics.median(ts)


def event_time(fn, iters=10):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


def weight_sets(k, n, wdt, gs, g):
    """Enough random quantised weight sets [(w, scale)] to exceed the L2 together."""
    wbytes = n * k // (2 if wdt == "int4" else 1) + 4 * n * (1 if gs < 0 else k // gs)
    cnt = max(2, math.ceil(2 * L2 / wbytes))
    sets = []
    for _ in range(cnt):
        w = torch.randint(-128, 128, (n, k // 2 if wdt == "int4" else k), device="cuda", dtype=torch.int8, generator=g)
        s = torch.rand((n,) if gs < 0 else (k // gs, n), device="cuda", generator=g) * 1e-2
        sets.append((w, s))
    return sets, wbytes


def bench_kernel(g):
    E = ext()
    rows = []
    for model, shapes in SHAPES.items():
        for name, k, n in shapes:
            bbytes = 2 * k * n
            bsets = [torch.randn(k, n, device="cuda", generator=g).to(torch.bfloat16) for _ in range(max(2, math.ceil(2 * L2 / bbytes)))]
            qsets = {v: weight_sets(k, n, *v, g) for v in VARIANTS}
            for m in (1, 16, 64):
                x = (torch.randn(m, k, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
                row = {"model": model, "layer": name, "k": k, "n": n, "m": m}
                it = [0]

                def bf16():
                    it[0] += 1
                    KG.linear(x, bsets[it[0] % len(bsets)])

                t = graph_time(bf16)
                row["bf16_us"] = round(t * 1e3, 2)
                row["bf16_GBps"] = round(bbytes / t / 1e6, 1)
                row["bf16_of_peak"] = round(bbytes / t / 1e-3 / HBM, 3)
                for (wdt, gs) in VARIANTS:
                    sets, wbytes = qsets[(wdt, gs)]
                    key = f"{wdt}_{'pc' if gs < 0 else f'g{gs}'}"

                    def wo(sets=sets, wdt=wdt, gs=gs):
                        it[0] += 1
                        w, s = sets[it[0] % len(sets)]
                        E.weight_only_gemm(x, w, s, None, wdt == "int4", gs)

                    t = graph_time(wo)
                    row[f"{key}_us"] = round(t * 1e3, 2)
                    row[f"{key}_GBps"] = round(wbytes / t / 1e6, 1)
                    row[f"{key}_of_peak"] = round(wbytes / t / 1e-3 / HBM, 3)
                    row[f"{key}_speedup_vs_bf16"] = round(row["bf16_us"] / row[f"{key}_us"], 2)
                for wdt in ("int8", "int4"):
                    for gs in (64, 128):
                        row[f"{wdt}_g{gs}_cost_vs_pc"] = round(row[f"{wdt}_g{gs}_us"] / row[f"{wdt}_pc_us"], 3)
                rows.append(row)
                print(json.dumps(row), flush=True)
            del bsets, qsets
            torch.cuda.empty_cache()
    return rows


def bench_dequant(g):
    E = ext()
    rows = []
    k, n = 5120, 27648
    for wdt, gs in (("int8", -1), ("int4", 128)):
        w = torch.randint(-128, 128, (n, k // 2 if wdt == "int4" else k), device="cuda", dtype=torch.int8, generator=g)
        s = torch.rand((n,) if gs < 0 else (k // gs, n), device="cuda", generator=g) * 1e-2
        arms = {"kernel": lambda: E.weight_dequantize(w, s, wdt == "int4", gs, torch.bfloat16),
                "torch": lambda: Q._dequantize_torch(w, s, wdt == "int4", torch.bfloat16, gs)}
        row = {"k": k, "n": n, "weights": wdt, "group_size": gs, "bitwise_equal": bool(torch.equal(arms["kernel"](), arms["torch"]()))}
        for arm, fn in arms.items():
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = fn()
            torch.cuda.synchronize()
            row[f"{arm}_peak_MB"] = round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)
            del out
            t = event_time(fn)
            row[f"{arm}_ms"] = round(t, 3)
        row["speedup"] = round(row["torch_ms"] / row["kernel_ms"], 2)
        row["kernel_GBps"] = round((w.numel() + s.numel() * 4 + 2 * k * n) / row["kernel_ms"] / 1e6, 1)
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def bench_crossover(g):
    E = ext()
    rows = []
    for name, k, n in (SHAPES["7b"][2], SHAPES["13b"][3]):
        for wdt, gs in (("int8", -1), ("int4", 128)):
            sets, _ = weight_sets(k, n, wdt, gs, g)
            for m in (64, 128, 256):
                x = (torch.randn(m, k, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
                it = [0]

                def in_sm():
                    it[0] += 1
                    w, s = sets[it[0] % len(sets)]
                    for r in range(0, m, 64):
                        E.weight_only_gemm(x[r:r + 64], w, s, None, wdt == "int4", gs)

                def dq_gemm():
                    it[0] += 1
                    w, s = sets[it[0] % len(sets)]
                    KG.linear(x, E.weight_dequantize(w, s, wdt == "int4", gs, torch.bfloat16))

                row = {"layer": name, "k": k, "n": n, "weights": wdt, "group_size": gs, "m": m,
                       "in_sm_us": round(graph_time(in_sm) * 1e3, 1), "dequant_gemm_us": round(graph_time(dq_gemm) * 1e3, 1)}
                rows.append(row)
                print(json.dumps(row), flush=True)
            del sets
            torch.cuda.empty_cache()
    return rows


def bench_engine(steps, rounds):
    from paddle_b200 import models

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.LlamaConfig(vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32,
                                 num_key_value_heads=32, max_position_embeddings=4096)
        ref = models.LlamaForCausalLM(cfg)
        ref.eval()
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    rows = []
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, cfg.vocab_size, (128,), generator=g).tolist() for _ in range(64)]
    for label, algo, gs in (("bf16", None, None), ("int8_pc", "weight_only_int8", -1), ("int4_g128", "weight_only_int4", 128)):
        m = ref if algo is None else models.quantize_weights(copy.deepcopy(ref), algo, gs)
        torch.cuda.synchronize()
        for batch in (1, 16, 64):
            eng = models.LLMEngine(m, num_blocks=batch * ((128 + steps * rounds + 32) // 16 + 1), block_size=16, max_running=batch)
            for p in prompts[:batch]:
                eng.add_request(p, steps * rounds + 16)
            eng.step()                                               # every prompt prefills in this step
            for _ in range(3):
                eng.step()                                           # warm-up decode steps
            meds = []
            for _ in range(rounds):
                ts = []
                for _ in range(steps):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    eng.step()
                    torch.cuda.synchronize()
                    ts.append((time.perf_counter() - t0) * 1e3)
                meds.append(statistics.median(ts))
            row = {"weights": label, "running": batch, "step_ms_median": round(statistics.median(meds), 2), "step_ms_min": round(min(meds), 2),
                   "step_ms_max": round(max(meds), 2), "rounds": rounds, "steps_per_round": steps}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del eng
            torch.cuda.empty_cache()
        if m is not ref:
            del m
            torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernel,dequant,crossover,engine")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_weight_only_serving.py measures on the GPU; no CUDA device is visible")
    torch.set_grad_enabled(False)
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"gpu": gpu_identity()}
    print(json.dumps(res["gpu"]), flush=True)
    parts = a.parts.split(",")
    if "kernel" in parts:
        res["kernel"] = bench_kernel(g)
    if "dequant" in parts:
        res["dequant"] = bench_dequant(g)
    if "crossover" in parts:
        res["crossover"] = bench_crossover(g)
    if "engine" in parts:
        res["engine"] = bench_engine(a.steps, a.rounds)
    res["gpu_after"] = gpu_identity()
    print(json.dumps(res["gpu_after"]), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
