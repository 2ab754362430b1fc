"""The qkv prologue of block_multihead_attention fused into the paged cache write, against the unfused sequence the same call would need
otherwise, on Llama-style GQA shapes: 32 query / 8 KV heads of 128, bf16 compute, block 64.

  fused    one `paged_kv_cache_write` launch: int32 dequantization (int32 input), bias, neox rotary, the processed rows written back and the
           K / V rows stored (bf16 copy or int8 quantization)
  unfused  torch dequantization (int32 input), torch bias add, `apply_rope_packed` (the models' rotary kernel), then the indexed scatter
           (bf16 cache) or `paged_kv_cache_write` (int8 cache), positions found on the device as block_attention finds them

Cases: 8192 prefill tokens of one sequence, and 256 decode rows with 2048 cached tokens each; bf16 and int32 qkv; bf16 and int8 caches.
Also output quantization of 8192 x 4096 bf16 to int8: `attention_out_quant` against the same rule in torch ops.

Times are medians of CUDA-event times over 20 runs after 5 warm-up runs; the two arms alternate over --rounds rounds and the median round
is reported.  GB/s counts the bytes the work needs (the rows read, the processed rows and the cache rows written), the same for both arms.
Outputs are compared between the arms.  The card's name and power limit are printed with the numbers.

  python scripts/bench_qkv_prologue.py [--rounds N] [--json FILE]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_paged_prefill import gpu_identity, timeit  # noqa: E402
from paddle_b200._build import ext  # noqa: E402
from paddle_b200.incubate.nn import paged_attention as PA  # noqa: E402
from paddle_b200.kernels import rope as R  # noqa: E402

NH, NKV, D, BS = 32, 8, 128, 64
W = (NH + 2 * NKV) * D


def make_case(kind, qkv_dtype, cache, g):
    if kind == "prefill":
        specs = [(8192, 0, 8192)]
    else:
        specs = [(0, 2048, 1)] * 256
    enc = torch.tensor([s[0] for s in specs], dtype=torch.int32, device="cuda")
    dec = torch.tensor([s[1] for s in specs], dtype=torch.int32, device="cuda")
    now = torch.tensor([s[2] for s in specs], dtype=torch.int32, device="cuda")
    cu = torch.zeros(len(specs) + 1, dtype=torch.int32, device="cuda")
    cu[1:] = torch.cumsum(now, 0)
    nblk = [((0 if e > 0 else d) + n + BS - 1) // BS for e, d, n in specs]
    bt = torch.randperm(sum(nblk), generator=g, device="cuda").to(torch.int32).reshape(len(specs), -1).contiguous()
    t = int(cu[-1])
    if qkv_dtype == "int32":
        qkv = torch.randint(-3000, 3000, (t, W), generator=g, device="cuda", dtype=torch.int32)
    else:
        qkv = (torch.randn(t, W, generator=g, device="cuda") * 0.5).to(torch.bfloat16)
    col_scale = torch.rand(W, generator=g, device="cuda") * 4e-4
    bias = (torch.randn(W, generator=g, device="cuda") * 0.1).to(torch.bfloat16)
    cos, sin = R.rope_tables(8192, D, 10000.0, device="cuda")      # every position of both cases
    cos2, sin2 = torch.cat([cos, cos], -1).contiguous(), torch.cat([sin, sin], -1).contiguous()
    kv_dt = torch.bfloat16 if cache == "bf16" else torch.int8
    kc = torch.zeros(sum(nblk), NKV, BS, D, device="cuda", dtype=kv_dt)
    vc = torch.zeros_like(kc)
    qs = torch.full((NKV,), 0.25, device="cuda")
    return dict(enc=enc, dec=dec, now=now, cu=cu, bt=bt, qkv=qkv, col_scale=col_scale, bias=bias, cos=cos, sin=sin, cos2=cos2, sin2=sin2,
                kc=kc, vc=vc, qs=qs, t=t)


def fused(c):
    x = torch.empty(c["t"], W, device="cuda", dtype=torch.bfloat16) if c["qkv"].dtype == torch.int32 else c["qkv"]
    scales = (None, None) if c["kc"].dtype == torch.bfloat16 else (c["qs"], c["qs"])
    ext().paged_kv_cache_write(c["qkv"], c["kc"], c["vc"], c["cu"], c["enc"], c["dec"], c["bt"], *scales, 1, 127.0, -127.0, qkv_out=x,
                               qkv_out_scale=c["col_scale"] if c["qkv"].dtype == torch.int32 else None, qkv_bias=c["bias"], rope_cos=c["cos2"],
                               rope_sin=c["sin2"], neox=True)
    return x


def unfused(c):
    qkv, cu, enc, dec, bt, t = c["qkv"], c["cu"], c["enc"], c["dec"], c["bt"], c["t"]
    x = (qkv.float() * c["col_scale"]).to(torch.bfloat16) if qkv.dtype == torch.int32 else qkv
    x = x + c["bias"]
    nseq = bt.shape[0]
    cu64 = cu.long()
    past = torch.where(enc > 0, torch.zeros_like(dec), dec).long()
    tok = torch.arange(t, device="cuda")
    seq_of = torch.bucketize(tok, cu64[1:], right=True).clamp(max=nseq - 1)
    pos = past[seq_of] + (tok - cu64[seq_of])
    x = R.apply_rope_packed(x.reshape(1, t, W), c["cos"], c["sin"], NH + NKV, NH + 2 * NKV, D, position_ids=pos[None], neox=True)
    x = x.as_subclass(torch.Tensor).reshape(t, W)
    if c["kc"].dtype == torch.bfloat16:
        rows = x.reshape(t, NH + 2 * NKV, D)
        blk, off = bt.long()[seq_of, pos // BS], pos % BS
        c["kc"][blk, :, off] = rows[:, NH:NH + NKV]
        c["vc"][blk, :, off] = rows[:, NH + NKV:]
    else:
        ext().paged_kv_cache_write(x, c["kc"], c["vc"], cu, enc, dec, bt, c["qs"], c["qs"], 1, 127.0, -127.0)
    return x


def prologue_bytes(c):
    inb = c["t"] * W * c["qkv"].element_size()
    return inb + c["t"] * W * 2 + 2 * c["t"] * NKV * D * c["kc"].element_size()


def compare(c):
    """max |fused - unfused| over the processed rows and the caches (the two rotary kernels may round differently in the last bit)."""
    kc0, vc0, qkv0 = c["kc"].clone(), c["vc"].clone(), c["qkv"].clone()
    a = fused(c).float()                                                   # a bf16 qkv is processed in place
    ka, va = c["kc"].float(), c["vc"].float()
    for k, v in (("kc", kc0), ("vc", vc0), ("qkv", qkv0)):
        c[k].copy_(v)
    b = unfused(c).float()
    kb, vb = c["kc"].float(), c["vc"].float()
    return {"rows_max_abs_diff": (a - b).abs().max().item(), "rows_max_abs": b.abs().max().item(),
            "cache_max_abs_diff": max((ka - kb).abs().max().item(), (va - vb).abs().max().item())}


def alternate(arms, rounds):
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timeit(fn))
    return {k: statistics.median(v) for k, v in times.items()}


def bench_prologue(kind, qkv_dtype, cache, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    c = make_case(kind, qkv_dtype, cache, g)
    check = compare(c)
    ms = alternate({"fused": lambda: fused(c), "unfused": lambda: unfused(c)}, rounds)
    nbytes = prologue_bytes(c)
    row = {"case": kind, "tokens": c["t"], "qkv": qkv_dtype, "cache": cache, **check}
    for k, v in ms.items():
        row[f"{k}_us"] = round(v * 1e3, 1)
        row[f"{k}_GBps"] = round(nbytes / v / 1e6, 1)
    row["speedup"] = round(ms["unfused"] / ms["fused"], 2)
    tol = 2 ** -7 * check["rows_max_abs"]
    assert check["rows_max_abs_diff"] <= tol and check["cache_max_abs_diff"] <= (1.0 if cache == "int8" else tol), row
    return row


def bench_out_quant(rounds, rows=8192, cols=4096):
    g = torch.Generator(device="cuda").manual_seed(1)
    o = (torch.randn(rows, cols, generator=g, device="cuda") * 2).to(torch.bfloat16)
    y = torch.empty(rows, cols, device="cuda", dtype=torch.int8)
    pro = PA.qkv_prologue_params(torch.zeros(1, 3 * D, dtype=torch.bfloat16, device="cuda"), 1, 1, D, out_scale=0.1)
    kernel = lambda: ext().attention_out_quant(o, y, 0.1, None, None, 1, 127.0, -127.0)   # noqa: E731
    kernel()
    want = PA._out_quant_ref(o, pro)
    assert torch.equal(y, want)
    ms = alternate({"kernel": kernel, "torch": lambda: PA._out_quant_ref(o, pro)}, rounds)
    nbytes = rows * cols * 3
    row = {"case": "out_quant", "rows": rows, "cols": cols, "bitwise_equal": True}
    for k, v in ms.items():
        row[f"{k}_us"] = round(v * 1e3, 1)
        row[f"{k}_GBps"] = round(nbytes / v / 1e6, 1)
    row["speedup"] = round(ms["torch"] / ms["kernel"], 2)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_qkv_prologue.py measures on the GPU; no CUDA device is visible")
    res = {"gpu": gpu_identity(), "prologue": [], "out_quant": None}
    print(json.dumps(res["gpu"]), flush=True)
    for kind in ("prefill", "decode"):
        for qkv_dtype in ("bf16", "int32"):
            for cache in ("bf16", "int8"):
                res["prologue"].append(bench_prologue(kind, qkv_dtype, cache, a.rounds))
                print(json.dumps(res["prologue"][-1]), flush=True)
    res["out_quant"] = bench_out_quant(a.rounds)
    print(json.dumps(res["out_quant"]), flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
