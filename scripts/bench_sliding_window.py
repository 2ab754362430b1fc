"""Sliding-window attention (W = 4096, Mistral-7B's attention shape: 32 query / 8 KV heads of 128, bf16, block_size 64) on the sm_90a kernels.

  decode   `decode_attention_paged`, batch 8 / 64, context 4k / 8k / 16k / 32k, windowed (window=4096) beside unwindowed, and unwindowed at
           context 4096.  A windowed call reads min(context, W) cache rows per sequence.
  verify   `decode_attention_paged_multi`: 5-token rows (k = 4 speculation) over the same contexts, batch 8 / 64.
  prefill  `attention_fwd_paged`: one 2048-token chunk over a cached prefix of 4k / 8k / 16k / 30k tokens, batch 1, windowed and not.
  capacity the number of concurrent generations (prompt 1024 + 31k new tokens) an 80 GB-class pool of 60000 blocks of 64 tokens holds
           at their final length, with and without the window: counted from LLMEngine's release rule, not timed.

Kernel times are medians of CUDA-event times (bench_paged_prefill.timeit).  The card's name and power limit are read in the same run.

  python scripts/bench_sliding_window.py [--parts decode,verify,prefill,capacity] [--json FILE]
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

NH, NKV, D, BS, W = 32, 8, 128, 64, 4096
CONTEXTS = (4096, 8192, 16384, 32768)


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def paged(batch, ctx, g):
    nblk = (ctx + BS - 1) // BS
    bt = torch.randperm(batch * nblk, device="cuda", generator=g).to(torch.int32).reshape(batch, nblk).contiguous()
    kc = (torch.randn(batch * nblk, NKV, BS, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    return bt, kc, torch.randn_like(kc)


def bench_decode(g):
    rows, scale = [], 1.0 / math.sqrt(D)
    for batch in (8, 64):
        for ctx in CONTEXTS:
            bt, kc, vc = paged(batch, ctx, g)
            q = torch.randn(batch, NH, D, device="cuda", generator=g).to(torch.bfloat16)
            lens = i32([ctx] * batch)
            r = {"batch": batch, "context": ctx}
            for name, w in (("full_us", 0), ("window_us", W)):
                r[name] = round(BP.timeit(lambda: ext().decode_attention_paged(q, kc, vc, lens, bt, scale, window=w)) * 1e3, 1)
            rows.append(r)
            del bt, kc, vc
    return rows


def bench_verify(g):
    rows, scale, n = [], 1.0 / math.sqrt(D), 5
    for batch in (8, 64):
        for ctx in CONTEXTS:
            bt, kc, vc = paged(batch, ctx + n, g)
            q = torch.randn(batch * n, NH, D, device="cuda", generator=g).to(torch.bfloat16)
            out = torch.empty(batch * n, NH * D, device="cuda", dtype=torch.bfloat16)
            cu, nq, past = i32([i * n for i in range(batch)]), i32([n] * batch), i32([ctx] * batch)
            r = {"batch": batch, "context": ctx}
            for name, w in (("full_us", 0), ("window_us", W)):
                r[name] = round(BP.timeit(lambda: ext().decode_attention_paged_multi(q, kc, vc, bt, cu, nq, past, scale, out, window=w)) * 1e3, 1)
            rows.append(r)
            del bt, kc, vc
    return rows


def bench_prefill(g):
    rows, scale, n = [], 1.0 / math.sqrt(D), 2048
    for past in (4096, 8192, 16384, 30720):
        bt, kc, vc = paged(1, past + n, g)
        q = torch.randn(n, NH, D, device="cuda", generator=g).to(torch.bfloat16)
        out = torch.empty(n, NH * D, device="cuda", dtype=torch.bfloat16)
        r = {"chunk": n, "prefix": past}
        for name, w in (("full_ms", 0), ("window_ms", W)):
            r[name] = round(BP.timeit(lambda: ext().attention_fwd_paged(q, kc, vc, bt, i32([0]), i32([n]), i32([past]), scale, out, window=w)), 3)
        rows.append(r)
        del bt, kc, vc
    return rows


def capacity(num_blocks=60000, prompt=1024, new=31 * 1024):
    """Generations of prompt + new tokens that fit the pool at their final length: all blocks, or the window's blocks plus the one being
    written (LLMEngine frees block j once (j + 1) * BS <= cached - W + 1)."""
    total = prompt + new
    full = -(-total // BS)
    dead = max(total - W + 1, 0) // BS
    windowed = -(-(total + 1) // BS) - dead
    return {"pool_blocks": num_blocks, "tokens_per_generation": total, "blocks_full": full, "blocks_windowed": windowed,
            "concurrent_full": num_blocks // full, "concurrent_windowed": num_blocks // windowed}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="decode,verify,prefill,capacity")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    parts = args.parts.split(",")
    res = {}
    if "capacity" in parts:
        res["capacity"] = capacity()
    if any(p in parts for p in ("decode", "verify", "prefill")):
        res["gpu"] = BP.gpu_identity()
        g = torch.Generator(device="cuda").manual_seed(0)
        for p, fn in (("decode", bench_decode), ("verify", bench_verify), ("prefill", bench_prefill)):
            if p in parts:
                res[p] = fn(g)
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
