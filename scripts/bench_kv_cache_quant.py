"""Quantized paged KV cache (int8 / fp8 e4m3) against a bf16 cache on Llama-2-7B attention shapes: 32 heads of 128, bf16 queries.

  decode   `decode_attention_paged`, batch 32, contexts 1k / 4k / 16k, block 64: microseconds, and cache bytes read per second against
           the 3.35 TB/s HBM3 data-sheet figure (the K and V rows of every context, which the kernel reads exactly once)
  prefill  `attention_fwd_paged`, one 2048-token chunk over 4k and 16k cached prefixes, block 64: the 8-bit kernel over the bf16 kernel
  write    8192 new tokens into the cache: `paged_kv_cache_write` (quantizing, one launch) against the bf16 indexed scatter that
           `block_attention` uses for 16-bit caches

Times are medians of CUDA-event times over 20 runs after 5 warm-up runs.  The card's name and power limit are printed with the numbers.

  python scripts/bench_kv_cache_quant.py [--quick] [--json FILE]
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_paged_prefill import causal_flops, gpu_identity, timeit  # noqa: E402
from paddle_b200._build import ext  # noqa: E402

NH, NKV, D, BS = 32, 32, 128, 64
HBM = 3.35e12
KINDS = {"bf16": torch.bfloat16, "int8": torch.int8, "fp8": torch.float8_e4m3fn}


def caches(kind, nblocks, g):
    dt = KINDS[kind]
    shape = (nblocks, NKV, BS, D)
    if dt == torch.int8:
        return [torch.randint(-127, 128, shape, generator=g, device="cuda", dtype=torch.int8) for _ in range(2)]
    return [(torch.randn(shape, generator=g, device="cuda") * (64 if dt == torch.float8_e4m3fn else 0.5)).to(dt) for _ in range(2)]


def dq_args(kind):
    if kind == "bf16":
        return {}
    s = torch.full((NKV,), 1.0 / 64, device="cuda")
    return {"k_dequant_scales": s, "v_dequant_scales": s}


def bench_decode(ctx, batch=32):
    g = torch.Generator(device="cuda").manual_seed(0)
    nblk = (ctx + BS - 1) // BS
    bt = torch.randperm(batch * nblk, device="cuda", generator=g).to(torch.int32).reshape(batch, nblk).contiguous()
    q = torch.randn(batch, NH, D, device="cuda", generator=g).to(torch.bfloat16)
    lens = torch.full((batch,), ctx, dtype=torch.int32, device="cuda")
    row = {"context": ctx, "batch": batch}
    for kind, dt in KINDS.items():
        kc, vc = caches(kind, batch * nblk, g)
        dq = dq_args(kind)
        ms = timeit(lambda: ext().decode_attention_paged(q, kc, vc, lens, bt, 1 / math.sqrt(D), **dq))
        nbytes = 2 * batch * ctx * NKV * D * kc.element_size()
        row[kind] = {"us": round(ms * 1e3, 1), "cache_GBps": round(nbytes / ms / 1e6, 1), "share_of_hbm": round(nbytes / ms / 1e-3 / HBM, 3)}
        del kc, vc
    row["int8_speedup"] = round(row["bf16"]["us"] / row["int8"]["us"], 3)
    row["fp8_speedup"] = round(row["bf16"]["us"] / row["fp8"]["us"], 3)
    return row


def bench_prefill(past, n=2048):
    g = torch.Generator(device="cuda").manual_seed(1)
    total = past + n
    nblk = (total + BS - 1) // BS
    bt = torch.randperm(nblk, device="cuda", generator=g).to(torch.int32).reshape(1, -1).contiguous()
    q = torch.randn(n, NH, D, device="cuda", generator=g).to(torch.bfloat16)
    out = torch.empty(n, NH * D, device="cuda", dtype=torch.bfloat16)
    i32 = lambda v: torch.tensor([v], dtype=torch.int32, device="cuda")   # noqa: E731
    cu, nq, pa = i32(0), i32(n), i32(past)
    flops = causal_flops([(past, n)])
    row = {"past": past, "new": n}
    for kind in KINDS:
        kc, vc = caches(kind, nblk, g)
        dq = dq_args(kind)
        ms = timeit(lambda: ext().attention_fwd_paged(q, kc, vc, bt, cu, nq, pa, 1 / math.sqrt(D), out, **dq))
        row[kind] = {"ms": round(ms, 3), "TFLOPs": round(flops / ms / 1e9, 1)}
    row["int8_over_bf16"] = round(row["bf16"]["ms"] / row["int8"]["ms"], 3)
    row["fp8_over_bf16"] = round(row["bf16"]["ms"] / row["fp8"]["ms"], 3)
    return row


def bench_write(t=8192):
    g = torch.Generator(device="cuda").manual_seed(2)
    nblk = (t + BS - 1) // BS
    qkv = torch.randn(t, (NH + 2 * NKV) * D, device="cuda", generator=g).to(torch.bfloat16)
    bt = torch.randperm(nblk, device="cuda", generator=g).to(torch.int32).reshape(1, -1).contiguous()
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    cu, enc, dec = i32(0, t), i32(t), i32(0)
    rows = qkv.reshape(t, NH + 2 * NKV, D)
    k, v = rows[:, NH:NH + NKV], rows[:, NH + NKV:]
    pos = torch.arange(t, device="cuda")
    blk, off = bt[0].long()[pos // BS], pos % BS
    kc16 = torch.zeros(nblk, NKV, BS, D, device="cuda", dtype=torch.bfloat16)
    vc16 = torch.zeros_like(kc16)

    def scatter():
        kc16[blk, :, off] = k
        vc16[blk, :, off] = v

    row = {"tokens": t, "bf16_scatter_us": round(timeit(scatter) * 1e3, 1)}
    s = torch.full((NKV,), 1.0 / 4, device="cuda")
    for kind in ("int8", "fp8"):
        kc = torch.zeros(nblk, NKV, BS, D, device="cuda", dtype=KINDS[kind])
        vc = torch.zeros_like(kc)
        bound = 127.0 if kind == "int8" else 448.0
        ms = timeit(lambda: ext().paged_kv_cache_write(qkv, kc, vc, cu, enc, dec, bt, s, s, 1, bound, -bound))
        row[f"{kind}_write_us"] = round(ms * 1e3, 1)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_kv_cache_quant.py measures on the GPU; no CUDA device is visible")
    res = {"gpu": gpu_identity(), "decode": [], "prefill": [], "write": None}
    print(json.dumps(res["gpu"]), flush=True)
    for ctx in ((1024, 4096) if a.quick else (1024, 4096, 16384)):
        res["decode"].append(bench_decode(ctx))
        print(json.dumps(res["decode"][-1]), flush=True)
    for past in ((4096,) if a.quick else (4096, 16384)):
        res["prefill"].append(bench_prefill(past))
        print(json.dumps(res["prefill"][-1]), flush=True)
    res["write"] = bench_write()
    print(json.dumps(res["write"]), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
