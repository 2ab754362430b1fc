"""Training attention at head_dim 64 on the sm_90a kernels (csrc/attention_d64_sm100.cu) against torch SDPA, bf16, causal.

  kernel   forward, backward (single pass and deterministic) and forward + backward on [B,S,H,64] tensors of about 16k tokens:
           TinyLlama (32 / 4 heads, S 2048, B 8), Llama-3.2-1B attention (32 / 8 heads, S 4096, B 4), GPT-350M (16 / 16 heads,
           S 2048, B 8).  SDPA runs on the same tensors as [B,H,S,D] views with enable_gqa.  TFLOP/s counts the causal half:
           4 B H S^2 D / 2 for the forward and 2.5 times that for the backward.
  masked   forward + backward at S 4096, B 4, 32 / 4 heads under a causal document mask (four documents of 1024) and a causal
           1024-token window: the own kernels with their column mask against SDPA with the dense boolean mask.
  e2e      training-step tokens/s of tinyllama_1b() (22 layers), bf16, AdamW, B 4 x S 2048, own kernels against
           FLAGS_b200_flash_attention=0 (SDPA), the arms alternated --rounds times; median and spread (min, max) per arm.

Kernel times are medians over --reps windows of --iters launches each, timed with CUDA events after warm-up.  The card's name and power
limit, and the SDPA kernels torch picked (from a profiler run of their own), are read in the same run.

  python scripts/bench_attention_d64.py [--parts kernel,masked,e2e] [--json FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import paddle_b200 as paddle  # noqa: E402
from paddle_b200._build import ext  # noqa: E402
from paddle_b200.kernels import attention as KAT  # noqa: E402

D = 64
SC = D ** -0.5
SHAPES = [("tinyllama", 8, 2048, 32, 4), ("llama3.2-1b", 4, 4096, 32, 8), ("gpt-350m", 8, 2048, 16, 16)]


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    name, power, clock = (x.strip() for x in r.stdout.strip().split(",")[:3])
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timeit(fn, iters=20, reps=5, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / iters)
    return statistics.median(ts)


def sdpa_kernels(fn):
    """Names of the CUDA kernels one fn() launches (which SDPA backend torch picked)."""
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({e.key for e in prof.key_averages() if e.device_type.name == "CUDA" and ("attention" in e.key.lower() or "fmha" in e.key.lower() or "flash" in e.key.lower())})


def _deterministic(on):
    paddle.set_flags({"FLAGS_cudnn_deterministic": on})


def tensors(b, s, h, hk, g):
    mk = lambda n: torch.randn(b, s, n, D, device="cuda", generator=g).to(torch.bfloat16)  # noqa: E731
    return mk(h), mk(hk), mk(hk), mk(h)


def bench_kernel():
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    E = ext()
    for name, b, s, h, hk in SHAPES:
        q, k, v, do = tensors(b, s, h, hk, g)
        fl = 4 * b * h * s * s * D / 2
        out, lse = E.attention_fwd(q, k, v, SC, True)
        own = {"fwd": timeit(lambda: E.attention_fwd(q, k, v, SC, True)),
               "bwd": timeit(lambda: E.attention_bwd(q, k, v, out, lse, do, SC, True))}
        _deterministic(True)
        own["bwd_det"] = timeit(lambda: E.attention_bwd(q, k, v, out, lse, do, SC, True))
        _deterministic(False)

        def own_step():
            o, l = E.attention_fwd(q, k, v, SC, True)
            return E.attention_bwd(q, k, v, o, l, do, SC, True)

        own["fwd_bwd"] = timeit(own_step)
        qt, kt, vt, dot = (t.transpose(1, 2) for t in (q, k, v, do))
        qg, kg, vg = (t.detach().requires_grad_(True) for t in (qt, kt, vt))
        sd_fwd = lambda: F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, enable_gqa=hk != h)  # noqa: E731
        o_sd = F.scaled_dot_product_attention(qg, kg, vg, is_causal=True, enable_gqa=hk != h)
        sd_bwd = lambda: torch.autograd.grad(o_sd, (qg, kg, vg), dot, retain_graph=True)  # noqa: E731

        def sd_step():
            o = F.scaled_dot_product_attention(qg, kg, vg, is_causal=True, enable_gqa=hk != h)
            return torch.autograd.grad(o, (qg, kg, vg), dot)

        sdpa = {"fwd": timeit(sd_fwd), "bwd": timeit(sd_bwd), "fwd_bwd": timeit(sd_step)}
        row = {"part": "kernel", "shape": name, "b": b, "s": s, "h": h, "hk": hk, "sdpa_kernels": sdpa_kernels(sd_step)}
        for key, t in own.items():
            f = fl if key == "fwd" else (2.5 * fl if key.startswith("bwd") else 3.5 * fl)
            row[f"own_{key}"] = {"ms": round(t, 3), "tflops": round(f / t / 1e9, 1)}
            sk = "bwd" if key.startswith("bwd") else key
            row[f"own_{key}"]["x_sdpa"] = round(sdpa[sk] / t, 2)
        for key, t in sdpa.items():
            f = fl if key == "fwd" else (2.5 * fl if key == "bwd" else 3.5 * fl)
            row[f"sdpa_{key}"] = {"ms": round(t, 3), "tflops": round(f / t / 1e9, 1)}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del q, k, v, do, qg, kg, vg, o_sd
    return rows


def bench_masked():
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1)
    b, s, h, hk = 4, 4096, 32, 4
    q, k, v, do = tensors(b, s, h, hk, g)
    keys = torch.arange(s, device="cuda")
    doc_end = (keys // 1024 + 1) * 1024
    masks = {"causal_document_4x1024": KAT.colmask_from_startend(doc_end.reshape(1, 1, s, 1).expand(b, 1, s, 1).int().contiguous(), True, s),
             "causal_window_1024": KAT.colmask_from_window(s, s, 1023, 0, True, q.device).expand(b, 1, s, 4).contiguous()}
    for name, cm in masks.items():
        qg, kg, vg = (t.detach().requires_grad_(True) for t in (q, k, v))

        def own_step():
            o = KAT.attention_colmask(qg, kg, vg, cm, causal=True).as_subclass(torch.Tensor)
            return torch.autograd.grad(o, (qg, kg, vg), do)

        vis = KAT.colmask_to_dense(cm, s) & torch.ones(s, s, dtype=torch.bool, device="cuda").tril()
        qt, kt, vt = (t.detach().transpose(1, 2).requires_grad_(True) for t in (q, k, v))
        dot = do.transpose(1, 2)

        def sd_step():
            o = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=vis, enable_gqa=True)
            return torch.autograd.grad(o, (qt, kt, vt), dot)

        t_own, t_sd = timeit(own_step, iters=10), timeit(sd_step, iters=5)
        row = {"part": "masked", "mask": name, "b": b, "s": s, "h": h, "hk": hk, "own_fwd_bwd_ms": round(t_own, 3),
               "sdpa_dense_mask_fwd_bwd_ms": round(t_sd, 3), "x_sdpa": round(t_sd / t_own, 2), "sdpa_kernels": sdpa_kernels(sd_step)}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del vis
    return rows


def bench_e2e(rounds, steps, warmup):
    from paddle_b200.models import LlamaForCausalLM, tinyllama_1b

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    paddle.seed(0)
    cfg = tinyllama_1b()
    model = LlamaForCausalLM(cfg)
    opt = paddle.optimizer.AdamW(1e-4, parameters=model.parameters(), weight_decay=0.1, multi_precision=True)
    b, s = 4, 2048
    ids = paddle.randint(0, cfg.vocab_size, [b, s + 1])

    def step():
        loss = model(ids[:, :-1], ids[:, 1:])
        loss.backward()
        opt.step()
        opt.clear_grad()
        return loss

    res = {"own": [], "sdpa": []}
    for r in range(rounds):
        for arm in ("own", "sdpa") if r % 2 == 0 else ("sdpa", "own"):
            paddle.set_flags({"FLAGS_b200_flash_attention": arm == "own"})
            for _ in range(warmup):
                step()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(steps):
                loss = step()
            float(loss.item())
            torch.cuda.synchronize()
            res[arm].append(b * s * steps / (time.perf_counter() - t0))
    paddle.set_flags({"FLAGS_b200_flash_attention": True})
    row = {"part": "e2e", "model": "tinyllama_1b (22 layers)", "b": b, "s": s, "steps": steps, "rounds": rounds}
    for arm, v in res.items():
        row[arm] = {"tokens_per_s_median": round(statistics.median(v), 1), "min": round(min(v), 1), "max": round(max(v), 1),
                    "runs": [round(x, 1) for x in v]}
    row["own_over_sdpa"] = round(row["own"]["tokens_per_s_median"] / row["sdpa"]["tokens_per_s_median"], 3)
    print(json.dumps(row), flush=True)
    paddle.set_default_dtype("float32")
    return [row]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernel,masked,e2e")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_attention_d64 needs a GPU"
    ident = gpu_identity()
    print(json.dumps(ident), flush=True)
    rows = []
    parts = args.parts.split(",")
    if "kernel" in parts:
        rows += bench_kernel()
    if "masked" in parts:
        rows += bench_masked()
    if "e2e" in parts:
        rows += bench_e2e(args.rounds, args.steps, args.warmup)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"identity": ident, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
