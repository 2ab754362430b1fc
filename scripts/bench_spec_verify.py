"""Attention for the verify rows of speculative decoding: n_q new tokens per sequence over a cached prefix in the paged KV cache.

Workloads: Llama-2-7B attention (32 query / 32 KV heads of 128) and a GQA shape (32 / 8), bf16 queries, block_size 64, batch 1 / 8 / 32,
contexts 1k / 4k / 16k and n_q 2 / 4 / 8 / 16 / 32 new tokens per sequence.  On the same rows it times
  multi    `decode_attention_paged_multi` (csrc/decode_attention.cu), the kernel block_attention uses for 2 <= n_q <= VERIFY_MAX
  prefill  `attention_fwd_paged` (csrc/attention_sm100.cu), the kernel it uses for longer chunks
  decode   n_q successive `decode_attention_paged` calls, one per new token over the growing prefix
with a bf16 cache, and with int8 and fp8 caches at context 4k.  n_q * (32 / KV heads) > 64 is beyond the multi kernel's row limit.
Times are medians of CUDA-event times over 10 runs after 3 warm-up runs; cache GB/s is the K and V bytes of every sequence's
context + n_q positions over the time, against the 3.35 TB/s HBM3 data-sheet figure.  The card's name and power limit are printed.

  python scripts/bench_spec_verify.py [--quick] [--json FILE]
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_paged_prefill as BP  # noqa: E402
from paddle_b200._build import ext  # noqa: E402

NH, D, BS = 32, 128, 64
HBM = 3.35e12
KINDS = {"bf16": torch.bfloat16, "int8": torch.int8, "fp8": torch.float8_e4m3fn}
BP.WARMUP, BP.ITERS = 3, 10


def caches(kind, shape, g):
    dt = KINDS[kind]
    if dt == torch.int8:
        return [torch.randint(-127, 128, shape, generator=g, device="cuda", dtype=torch.int8) for _ in range(2)]
    return [(torch.randn(shape, generator=g, device="cuda") * (64 if dt == torch.float8_e4m3fn else 0.5)).to(dt) for _ in range(2)]


def bench(nkv, batch, ctx, nqs, kinds):
    g = torch.Generator(device="cuda").manual_seed(0)
    nblk = (ctx + max(nqs) + BS - 1) // BS
    bt = torch.randperm(batch * nblk, device="cuda", generator=g).to(torch.int32).reshape(batch, nblk).contiguous()
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    scale = 1 / math.sqrt(D)
    rows = []
    for kind in kinds:
        kc, vc = caches(kind, (batch * nblk, nkv, BS, D), g)
        dq = {} if kind == "bf16" else {"k_dequant_scales": torch.full((nkv,), 1 / 64, device="cuda"),
                                        "v_dequant_scales": torch.full((nkv,), 1 / 64, device="cuda")}
        for nq in nqs:
            t = batch * nq
            q = torch.randn(t, NH, D, device="cuda", generator=g).to(torch.bfloat16)
            out = torch.empty(t, NH * D, device="cuda", dtype=torch.bfloat16)
            cu, n, past = i32([b * nq for b in range(batch)]), i32([nq] * batch), i32([ctx] * batch)
            qd = [q.reshape(batch, nq, NH, D)[:, j].contiguous() for j in range(nq)]
            lens = [i32([ctx + j + 1] * batch) for j in range(nq)]
            fns = {"prefill": lambda: ext().attention_fwd_paged(q, kc, vc, bt, cu, n, past, scale, out, **dq),
                   "decode": lambda: [ext().decode_attention_paged(qd[j], kc, vc, lens[j], bt, scale, **dq) for j in range(nq)]}
            if nq * (NH // nkv) <= 64:
                fns["multi"] = lambda: ext().decode_attention_paged_multi(q, kc, vc, bt, cu, n, past, scale, out, **dq)
            nbytes = 2 * batch * (ctx + nq) * nkv * D * kc.element_size()
            row = {"kv_heads": nkv, "batch": batch, "context": ctx, "n_q": nq, "cache": kind}
            for name in ("multi", "prefill", "decode"):
                if name in fns:
                    ms = BP.timeit(fns[name])
                    row[name] = {"us": round(ms * 1e3, 1), "cache_GBps": round(nbytes / ms / 1e6, 1), "share_of_hbm": round(nbytes / ms / 1e-3 / HBM, 3)}
            if "multi" in row:
                row["multi_speedup_vs_prefill"] = round(row["prefill"]["us"] / row["multi"]["us"], 2)
                row["multi_speedup_vs_decode"] = round(row["decode"]["us"] / row["multi"]["us"], 2)
            print(json.dumps(row), flush=True)
            rows.append(row)
        del kc, vc
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="one shape per KV-head count")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_spec_verify.py measures the GPU; there is nothing to measure without one"
    ident = BP.gpu_identity()
    print(json.dumps({"gpu": ident}), flush=True)
    rows = []
    batches, ctxs, nqs = ((8,), (4096,), (2, 8)) if args.quick else ((1, 8, 32), (1024, 4096, 16384), (2, 4, 8, 16, 32))
    for nkv in (32, 8):
        for batch in batches:
            for ctx in ctxs:
                rows += bench(nkv, batch, ctx, nqs, ["bf16"] + (["int8", "fp8"] if ctx == 4096 else []))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": ident, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
