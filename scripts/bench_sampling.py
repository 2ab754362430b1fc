"""Token sampling: the sm_90a sampling kernel (`sample_tokens`, csrc/sampling.cu) and LLMEngine's one sampling call per step.

Kernel part: bf16 logits, rows in {1, 8, 64, 256}, vocab in {32000, 128256, 152064}, modes greedy, top_k=50, top_p=0.9 and both
(temperature 1).  Three arms:

  kernel   one `sampling.sample` launch over the batch (per-row parameters already on the device)
  loop     the engine's earlier per-row loop: `_sample(logits[i:i+1], ...)` and `int(...)` per row, one device-to-host sync each
  batched  `_sample` over the whole batch: the same rule in torch ops (topk, full sort, softmax, cumsum, scatter, multinomial)

Times are medians of CUDA-event times (host gaps included: the loop arm waits on the host).  GB/s is rows * vocab * 2 bytes (one read
of the logits; top_k / top_p re-read the row from L2 once per radix digit) over the kernel time, against the 3.35 TB/s data-sheet HBM
bandwidth.

Engine part: a random-weight Llama-shaped model (bf16, hidden 1024, 4 layers, vocab 32000) with 64 running requests, all greedy or all
sampled (top_k=50, top_p=0.9).  Wall time of step() (it ends in the ids' device-to-host copy, so the device work is included) for the
new path and the swapped-in per-row loop, alternating in blocks of steps within one run; medians with the 10th-90th percentile spread.
The card's name and power limit are printed with the numbers.

  python scripts/bench_sampling.py [--quick] [--json FILE]
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_paged_prefill import gpu_identity  # noqa: E402
import paddle_b200 as paddle  # noqa: E402
from paddle_b200 import models  # noqa: E402
from paddle_b200.kernels import sampling  # noqa: E402
from paddle_b200.models.generation import _sample  # noqa: E402

MODES = {"greedy": (False, 0, 1.0), "top_k=50": (True, 50, 1.0), "top_p=0.9": (True, 0, 0.9), "both": (True, 50, 0.9)}
HBM = 3.35e12


def event_time(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3)
    return statistics.median(ts)


def kernel_cells(quick):
    out = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for vocab in (32000, 128256, 152064):
        for rows in ((1, 64) if quick else (1, 8, 64, 256)):
            x = (torch.randn(rows, vocab, generator=g, device="cuda") * 3).to(torch.bfloat16)
            for mode, (do_sample, k, p) in MODES.items():
                prm = [torch.full((rows,), 1.0 if do_sample else 0.0, device="cuda"), torch.full((rows,), k, dtype=torch.int32, device="cuda"),
                       torch.full((rows,), p, device="cuda"), torch.arange(rows, device="cuda"), torch.zeros(rows, dtype=torch.int64, device="cuda")]
                t_k = event_time(lambda: sampling.sample(x, *prm), 50)
                t_l = event_time(lambda: [int(_sample(x[i:i + 1], do_sample, 1.0, k, p)[0]) for i in range(rows)], 5 if rows > 8 else 10)
                t_b = event_time(lambda: _sample(x, do_sample, 1.0, k, p), 20)
                cell = {"vocab": vocab, "rows": rows, "mode": mode, "kernel_us": round(t_k, 1), "loop_us": round(t_l, 1),
                        "batched_torch_us": round(t_b, 1), "kernel_GBps": round(rows * vocab * 2 / t_k / 1e3, 1),
                        "share_of_hbm": round(rows * vocab * 2 / (t_k * 1e-6) / HBM, 3)}
                print(json.dumps(cell), flush=True)
                out.append(cell)
    return out


def old_rows(logits, rows):
    """The engine's sampling before the batched call: one _sample and one host read per row that yields a token."""
    return [int(_sample(logits[i:i + 1], s.do_sample, s.temperature, s.top_k, s.top_p)[0]) if s is not None else -1
            for i, s in enumerate(rows)]


def engine_cells(quick):
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    paddle.seed(0)
    cfg = models.llama_tiny(hidden_size=1024, intermediate_size=2816, num_attention_heads=8, num_key_value_heads=8, num_hidden_layers=4,
                            vocab_size=32000, max_position_embeddings=4096)
    m = models.LlamaForCausalLM(cfg)
    m.eval()
    paddle.set_default_dtype("float32")
    res = []
    block, rounds = (5, 4) if quick else (10, 8)
    for label, kw in (("greedy", {}), ("sampled", dict(do_sample=True, temperature=1.0, top_k=50, top_p=0.9))):
        eng = models.LLMEngine(m, num_blocks=64 * 24, block_size=16, max_running=64)
        g = torch.Generator().manual_seed(1)
        for _ in range(64):
            eng.add_request(torch.randint(1, cfg.vocab_size, (64,), generator=g).tolist(), 2 * block * rounds + 8, **kw)
        eng.step()                                                   # every prompt prefilled
        for _ in range(3):
            eng.step()
        new = eng._sample_rows
        times = {"batched_call": [], "per_row_loop": []}
        for r in range(rounds):
            for arm in (("batched_call", "per_row_loop") if r % 2 == 0 else ("per_row_loop", "batched_call")):
                eng._sample_rows = new if arm == "batched_call" else old_rows
                for _ in range(block):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    eng.step()
                    times[arm].append((time.perf_counter() - t0) * 1e3)
        assert len(eng.running) == 64
        for arm, ts in times.items():
            q = statistics.quantiles(ts, n=10)
            cell = {"requests": label, "arm": arm, "step_ms_median": round(statistics.median(ts), 2), "p10": round(q[0], 2),
                    "p90": round(q[-1], 2), "steps": len(ts)}
            print(json.dumps(cell), flush=True)
            res.append(cell)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampling.py needs a GPU")
    ident = gpu_identity()
    print(json.dumps(ident))
    kern = kernel_cells(a.quick)
    eng = engine_cells(a.quick)
    print(json.dumps(ident))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"gpu": ident, "kernel": kern, "engine": eng}, f, indent=1)


if __name__ == "__main__":
    main()
