"""Micro-benchmarks on the flagship shapes (Llama-2-7B, one 4096-token sequence per micro-batch): the persistent GEMM against
torch.matmul (cuBLAS) on every linear layer's forward, dX and dW shape, causal flash attention forward / backward against torch SDPA,
and the HBM-bound kernels against a device copy. Shares of peak use the H100 SXM data sheet (989 TFLOP/s dense bf16, 3.35 TB/s HBM3);
the card's name and power limit are printed with the numbers.

  python scripts/bench_kernels.py [all|gemm|attn|bw] [--quick] [--dump DIR] [--json FILE]

--quick   small shapes and few iterations (a fast end-to-end pass, e.g. under compute-sanitizer)
--dump    write every GEMM output and the attention outputs for seeded inputs as DIR/<name>.npy (16-bit outputs as their raw bits in
          int16), so that two builds can be compared bit for bit
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from paddle_b200._build import ext  # noqa: E402

PEAK_BF16_TFLOPS = 989.0   # H100 SXM data sheet, dense bf16, 700 W
PEAK_HBM_GBS = 3350.0

# (tag, M, N, K): forward (A [M,K], B = weight [in, out]); dX (b_is_nk: B = weight read as [N, K]); dW (a_is_km: A = X stored [K, M],
# B = dY [K, N] MN-major, accumulated into a bf16 gradient with epilogue 4, as the fused weight-gradient path does)
H, F, V, T = 4096, 11008, 32000, 4096
GEMMS = {
    "fwd": [("qkv", T, 3 * H, H), ("o", T, H, H), ("gate_up", T, 2 * F, H), ("down", T, H, F), ("lm_head", T, V, H)],
    "dx": [("qkv", T, H, 3 * H), ("o", T, H, H), ("gate_up", T, H, 2 * F), ("down", T, F, H), ("lm_head", T, H, V)],
    "dw": [("qkv", H, 3 * H, T), ("o", H, H, T), ("gate_up", H, 2 * F, T), ("down", F, H, T)],
}
QUICK_GEMMS = {"fwd": [("small", 256, 384, 192)], "dx": [("small", 256, 192, 384)], "dw": [("small", 192, 384, 256)]}

E = None
ITERS, WARMUP = 20, 5
_flush = None


def gpu_identity():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        name, power, clock = (x.strip() for x in r.stdout.strip().split(",")[:3])
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "note": "nvidia-smi unavailable"}


def timeit(fn, iters=None, warmup=None):
    """Median over `iters` launches of CUDA-event time; L2 is flushed before each."""
    iters, warmup = iters or ITERS, warmup or WARMUP
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        _flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def seeded(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(torch.bfloat16)


def save(dump, name, t):
    if not dump:
        return
    import numpy as np

    t = t.detach().contiguous()
    arr = t.view(torch.int16).cpu().numpy() if t.element_size() == 2 else t.cpu().numpy()
    np.save(os.path.join(dump, name + ".npy"), arr.astype(np.int16 if t.element_size() == 2 else np.float32))


def gemm_bench(quick, dump):
    rows = []
    seed = 0
    for mode, shapes in (QUICK_GEMMS if quick else GEMMS).items():
        for (tag, m, n, k) in shapes:
            seed += 1
            if mode == "fwd":
                A, B = seeded((m, k), seed), seeded((k, n), seed + 1000)
                run = lambda: E.gemm(A, B)                                                       # noqa: E731
                ref = lambda: torch.matmul(A, B)                                                 # noqa: E731
            elif mode == "dx":
                A, B = seeded((m, k), seed), seeded((n, k), seed + 1000)
                run = lambda: E.gemm(A, B, None, False, True)                                    # noqa: E731
                ref = lambda: torch.matmul(A, B.t())                                             # noqa: E731
            else:
                A, B = seeded((k, m), seed), seeded((k, n), seed + 1000)
                G0 = seeded((m, n), seed + 2000, 16.0)
                G = G0.clone()
                run = lambda: E.gemm(A, B, None, True, False, 4, G)                              # noqa: E731
                ref = lambda: G.addmm_(A.t(), B)                                                 # noqa: E731
            out = run()
            torch.cuda.synchronize()
            save(dump, f"gemm_{mode}_{tag}", out)
            t_mine = timeit(run)
            t_ref = timeit(ref)
            fl = 2.0 * m * n * k
            r = dict(kernel="gemm", mode=mode, tag=tag, m=m, n=n, k=k, ms=round(t_mine, 4), tflops=round(fl / t_mine / 1e9, 1),
                     share_of_989=round(fl / t_mine / 1e9 / PEAK_BF16_TFLOPS, 3), torch_ms=round(t_ref, 4), torch_tflops=round(fl / t_ref / 1e9, 1))
            print(json.dumps(r), flush=True)
            rows.append(r)
            del A, B, out
            if mode == "dw":
                del G, G0
    return rows


def attn_bench(quick, dump):
    """Causal flash attention of one 4096-token sequence, 32 heads of 128 (Llama-2-7B), against torch SDPA."""
    import torch.nn.functional as tnf

    b, s, h, d = (1, 256, 4, 128) if quick else (1, 4096, 32, 128)
    q, k, v = (seeded((b, s, h, d), 100 + i) for i in range(3))
    flops = 4.0 * b * h * s * s * d * 0.5
    out, lse = E.attention_fwd(q, k, v, d ** -0.5, True)
    g = seeded(out.shape, 104)
    grads = E.attention_bwd(q, k, v, out, lse, g, d ** -0.5, True)
    torch.cuda.synchronize()
    save(dump, "attn_fwd_out", out)
    save(dump, "attn_fwd_lse", lse)
    for name, t in zip(("dq", "dk", "dv"), grads):
        save(dump, f"attn_bwd_{name}", t)
    t = timeit(lambda: E.attention_fwd(q, k, v, d ** -0.5, True))
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    t_lib = timeit(lambda: tnf.scaled_dot_product_attention(qt, kt, vt, is_causal=True))
    rows = [dict(kernel="flash_attn_fwd", b=b, s=s, h=h, d=d, causal=True, ms=round(t, 4), tflops=round(flops / t / 1e9, 1),
                 share_of_989=round(flops / t / 1e9 / PEAK_BF16_TFLOPS, 3), torch_ms=round(t_lib, 4), torch_tflops=round(flops / t_lib / 1e9, 1))]
    print(json.dumps(rows[-1]), flush=True)
    tb = timeit(lambda: E.attention_bwd(q, k, v, out, lse, g, d ** -0.5, True))
    qr, kr, vr = (x.detach().requires_grad_(True) for x in (qt, kt, vt))
    o2 = tnf.scaled_dot_product_attention(qr, kr, vr, is_causal=True)
    g2 = g.transpose(1, 2)
    tb_lib = timeit(lambda: torch.autograd.grad(o2, (qr, kr, vr), g2, retain_graph=True))
    rows.append(dict(kernel="flash_attn_bwd", b=b, s=s, h=h, d=d, causal=True, ms=round(tb, 4), tflops=round(2.5 * flops / tb / 1e9, 1),
                     share_of_989=round(2.5 * flops / tb / 1e9 / PEAK_BF16_TFLOPS, 3), torch_ms=round(tb_lib, 4),
                     torch_tflops=round(2.5 * flops / tb_lib / 1e9, 1)))
    print(json.dumps(rows[-1]), flush=True)
    return rows


def bw_bench(quick):
    rows = []
    tok = 512 if quick else T
    x = torch.randn(tok, H, device="cuda", dtype=torch.bfloat16)
    w = torch.ones(H, device="cuda", dtype=torch.bfloat16)
    t = timeit(lambda: E.rms_norm_fwd(x, None, w, None, 1e-6))
    rows.append(dict(kernel="rms_norm_fwd", ms=round(t, 4), gbs=round(2 * x.numel() * 2 / t / 1e6, 1)))
    y, rstd, _ = E.rms_norm_fwd(x, None, w, None, 1e-6)
    t = timeit(lambda: E.rms_norm_bwd(y, x, w, rstd))
    rows.append(dict(kernel="rms_norm_bwd", ms=round(t, 4), gbs=round(3 * x.numel() * 2 / t / 1e6, 1)))
    gt = torch.randn(tok, F, device="cuda", dtype=torch.bfloat16)
    u = torch.randn_like(gt)
    t = timeit(lambda: E.swiglu_fwd(gt, u))
    rows.append(dict(kernel="swiglu_fwd", ms=round(t, 4), gbs=round(3 * gt.numel() * 2 / t / 1e6, 1)))
    lg = torch.randn(tok, V, device="cuda", dtype=torch.bfloat16)
    lab = torch.randint(0, V, (tok,), device="cuda")
    t = timeit(lambda: E.softmax_ce_fwd(lg, lab, -100))
    rows.append(dict(kernel="softmax_ce_fwd", ms=round(t, 4), gbs=round(lg.numel() * 2 / t / 1e6, 1)))
    n = 1 << (20 if quick else 28)
    p = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    gr = torch.randn(n, device="cuda", dtype=torch.bfloat16)
    ms_ = torch.zeros(n, device="cuda")
    m_ = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    v_ = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    t = timeit(lambda: E.adamw_step(p, gr, ms_, m_, v_, 1e-3, 0.9, 0.95, 1e-8, 0.1, 1, None, 0.0, None, None), iters=5, warmup=2)
    rows.append(dict(kernel="adamw(bf16 p/g/m/v + fp32 master)", ms=round(t, 4), gbs=round(n * (2 + 2 + 4 + 4 + 2 * 2 + 2 * 2) / t / 1e6, 1)))
    a = torch.empty(n * 2, device="cuda", dtype=torch.bfloat16)
    b = torch.empty_like(a)
    t = timeit(lambda: b.copy_(a), iters=5, warmup=2)
    rows.append(dict(kernel="torch copy (ref)", ms=round(t, 4), gbs=round(2 * a.numel() * 2 / t / 1e6, 1)))
    for r in rows:
        r["share_of_3350_gbs"] = round(r["gbs"] / PEAK_HBM_GBS, 3)
        print(json.dumps(r), flush=True)
    return rows


def main():
    global E, ITERS, WARMUP, _flush
    ap = argparse.ArgumentParser()
    ap.add_argument("which", nargs="?", default="all", choices=("all", "gemm", "attn", "bw"))
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--dump", default="", metavar="DIR")
    ap.add_argument("--json", default="", metavar="FILE", help="also write every row to FILE")
    args = ap.parse_args()
    E = ext()
    if args.quick:
        ITERS, WARMUP = 3, 1
    _flush = torch.empty((4 if args.quick else 256) << 20, dtype=torch.uint8, device="cuda")
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
    out = {"gpu": gpu_identity(), "peaks": {"bf16_tflops": PEAK_BF16_TFLOPS, "hbm_gbs": PEAK_HBM_GBS, "source": "H100 SXM data sheet"}}
    print(json.dumps(out["gpu"]), flush=True)
    if args.which in ("all", "gemm"):
        out["gemm"] = gemm_bench(args.quick, args.dump)
    if args.which in ("all", "attn"):
        out["attn"] = attn_bench(args.quick, args.dump)
    if args.which in ("all", "bw"):
        out["bw"] = bw_bench(args.quick)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
