"""int8 activations on the GPU: the int8 wgmma GEMM against the bf16 GEMM and the weight-only int8 routes, the per-token quantizer, and one
8192-token LLMEngine prefill step of a Llama-2-7B-shaped model with bf16, weight-only int8 and llm.int8 (threshold inf) weights.

  gemm       Llama-2-7B and 13B projection shapes (qkv, o, gate_up, down), m = 16 / 64 / 256 / 1024 / 4096 rows.  Arms: int8 x int8 with the
             int32 epilogue and with the dequantising bf16 epilogue (`gemm_int8`, `gemm_int8_dequant`), the bf16 `kernels.gemm`, and the
             weight-only int8 routes of `weight_only_linear` (the in-SM kernel for m <= 64, dequantise + bf16 GEMM above).  Each arm rotates
             through enough weight sets to exceed the 50 MB L2; calls are captured into one CUDA graph (20 calls) and replayed, the median of
             5 replays is reported per call.  TOPS = 2 m n k / time.
  quant      the per-token quantizer on [m, k] bf16, median CUDA-event time of 10 runs; GB/s counts x read, q written and the scales.
  engine     a random-weight Llama-2-7B-shaped model (32 layers), 8 prompts of 1024 tokens prefilled in one step; the step is timed on the
             host between device synchronizes, `--rounds` times after one warm-up, median and spread reported.

The card's name and power limit are read in the same run and printed with the numbers.

  python scripts/bench_llm_int8.py [--parts gemm,quant,engine] [--rounds N] [--json FILE]
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
from bench_weight_only_serving import L2, SHAPES, event_time, graph_time  # noqa: E402
import paddle_b200 as paddle  # noqa: E402
from paddle_b200._build import ext  # noqa: E402
from paddle_b200.kernels import gemm as KG  # noqa: E402

ROWS = (16, 64, 256, 1024, 4096)


def bench_gemm(g):
    E = ext()
    rows = []
    for model, shapes in SHAPES.items():
        for name, k, n in shapes:
            cnt = max(2, math.ceil(2 * L2 / (n * k)))
            bsets = [torch.randn(k, n, device="cuda", generator=g).to(torch.bfloat16) for _ in range(max(2, math.ceil(2 * L2 / (2 * n * k))))]
            qsets = [(torch.randint(-128, 128, (n, k), device="cuda", dtype=torch.int8, generator=g),
                      torch.rand(n, device="cuda", generator=g) * 1e-2) for _ in range(cnt)]
            for m in ROWS:
                x = (torch.randn(m, k, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
                xq = torch.randint(-128, 128, (m, k), device="cuda", dtype=torch.int8, generator=g)
                rs = torch.rand(m, device="cuda", generator=g) * 1e-2
                it = [0]

                def nxt(sets):
                    it[0] += 1
                    return sets[it[0] % len(sets)]

                def int8_bf16():
                    w, s = nxt(qsets)
                    E.gemm_int8_dequant(xq, w, rs, s, None, torch.bfloat16)

                arms = {"bf16": lambda: KG.gemm(x, nxt(bsets)),
                        "int8_i32": lambda: E.gemm_int8(xq, nxt(qsets)[0]),
                        "int8_bf16": int8_bf16}
                if m <= 64:
                    arms["wo_int8_in_sm"] = lambda: E.weight_only_gemm(x, *nxt(qsets), None, False, -1)
                arms["wo_int8_dequant_gemm"] = lambda: KG.gemm(x, E.weight_dequantize(*nxt(qsets), False, -1, torch.bfloat16))
                row = {"model": model, "layer": name, "m": m, "n": n, "k": k}
                for arm, fn in arms.items():
                    t = graph_time(fn)
                    row[f"{arm}_us"] = round(t * 1e3, 2)
                    row[f"{arm}_TOPS"] = round(2 * m * n * k / t / 1e9, 1)
                row["int8_bf16_speedup_vs_bf16"] = round(row["bf16_us"] / row["int8_bf16_us"], 2)
                rows.append(row)
                print(json.dumps(row), flush=True)
            del bsets, qsets
            torch.cuda.empty_cache()
    return rows


def bench_quant(g):
    E = ext()
    rows = []
    for m, k in ((1024, 4096), (8192, 4096), (8192, 11008)):
        x = torch.randn(m, k, device="cuda", generator=g).to(torch.bfloat16)
        t = event_time(lambda: E.quantize_int8_rows(x, None))
        row = {"m": m, "k": k, "ms": round(t, 4), "GBps": round((3 * m * k + 4 * m) / t / 1e6, 1)}
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def bench_engine(rounds):
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
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, cfg.vocab_size, (1024,), generator=g).tolist() for _ in range(8)]
    rows = []
    for label, algo in (("bf16", None), ("weight_only_int8", "weight_only_int8"), ("llm.int8", "llm.int8")):
        if algo is None:
            m = ref
        elif algo == "llm.int8":
            m = models.quantize_weights(copy.deepcopy(ref), algo, threshold=float("inf"))
        else:
            m = models.quantize_weights(copy.deepcopy(ref), algo)
        ts = []
        for r in range(rounds + 1):
            eng = models.LLMEngine(m, num_blocks=8192 // 16 + 64, block_size=16, max_running=8, max_batch_tokens=8192)
            for p in prompts:
                eng.add_request(p, 1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.step()                                                   # all 8192 prompt tokens in this step
            torch.cuda.synchronize()
            if r:
                ts.append((time.perf_counter() - t0) * 1e3)
            del eng
        row = {"weights": label, "prefill_tokens": 8192, "step_ms_median": round(statistics.median(ts), 2), "step_ms_min": round(min(ts), 2),
               "step_ms_max": round(max(ts), 2), "rounds": rounds}
        rows.append(row)
        print(json.dumps(row), flush=True)
        if m is not ref:
            del m
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="gemm,quant,engine")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_llm_int8.py measures on the GPU; no CUDA device is visible")
    torch.set_grad_enabled(False)
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"gpu": gpu_identity()}
    print(json.dumps(res["gpu"]), flush=True)
    parts = a.parts.split(",")
    if "gemm" in parts:
        res["gemm"] = bench_gemm(g)
    if "quant" in parts:
        res["quant"] = bench_quant(g)
    if "engine" in parts:
        res["engine"] = bench_engine(a.rounds)
    res["gpu_after"] = gpu_identity()
    print(json.dumps(res["gpu_after"]), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
