"""Prefill attention over the paged KV cache (`attention_fwd_paged`, csrc/attention_sm100.cu) on Llama-2-7B attention shapes: 32 heads
of 128, bf16.  Chunks of 512 and 2048 new tokens over cached prefixes of 0, 4096 and 16384 tokens, block_size 16 and 64, and a batch
of 16 fresh 512-token prompts.  Compared against

  dense         the own dense kernel (`attention_fwd`, causal) on the same K / V already contiguous: the ceiling
  gather+dense  gathering K / V out of the block table into contiguous tensors, then the dense kernel: the obvious alternative
  colmask       (16-prompt batch only) the earlier route for fresh prompts: the batch packed into one causal sequence with a padded
                copy of q / k / v and a per-document column mask, every CTA walking every earlier prompt's key tiles

Times are medians of CUDA-event times; TFLOP/s count the causal work from the shapes (4 * D flops per visible (query, key) pair and
head).  The card's name and power limit are printed with the numbers.

  python scripts/bench_paged_prefill.py [--quick] [--json FILE]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from paddle_b200._build import ext  # noqa: E402
from paddle_b200.kernels import attention as KAT  # noqa: E402

NH, NKV, D = 32, 32, 128
ITERS, WARMUP = 20, 5


def gpu_identity():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=20)
        name, power, clock = (x.strip() for x in r.stdout.strip().split(",")[:3])
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": None, "note": "nvidia-smi unavailable"}


def timeit(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(ITERS):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def causal_flops(seqs):
    """seqs: [(past, n)]: new row i sees past + i + 1 keys."""
    pairs = sum(n * past + n * (n + 1) // 2 for past, n in seqs)
    return 4.0 * D * NH * pairs


def make_case(seqs, bs, seed=0):
    """A paged cache holding every sequence's past + new tokens (shuffled blocks), the packed q rows, and the same K / V contiguous."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    need = [(past + n + bs - 1) // bs for past, n in seqs]
    nblocks = sum(need)
    perm = torch.randperm(nblocks, device="cuda", generator=g).to(torch.int32)
    bt = torch.zeros(len(seqs), max(need), dtype=torch.int32, device="cuda")
    kc = torch.empty(nblocks, NKV, bs, D, dtype=torch.bfloat16, device="cuda")
    vc = torch.empty_like(kc)
    Ks, Vs, o = [], [], 0
    for i, (past, n) in enumerate(seqs):
        bt[i, :need[i]] = perm[o:o + need[i]]
        o += need[i]
        total = past + n
        K = (torch.randn(total, NKV, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
        V = (torch.randn(total, NKV, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
        pos = torch.arange(total, device="cuda")
        blk = bt[i].long()[pos // bs]
        kc[blk, :, pos % bs] = K
        vc[blk, :, pos % bs] = V
        Ks.append(K)
        Vs.append(V)
    t = sum(n for _, n in seqs)
    qkv = (torch.randn(t, (NH + 2 * NKV) * D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    q = qkv.view(t, NH + 2 * NKV, D)[:, :NH]
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    cu = i32([0] + [sum(n for _, n in seqs[:i + 1]) for i in range(len(seqs) - 1)])
    return dict(q=q, kc=kc, vc=vc, bt=bt, cu=cu, n=i32([n for _, n in seqs]), past=i32([p for p, _ in seqs]), K=Ks, V=Vs, t=t)


def bench_case(label, seqs, bs, colmask=False):
    c = make_case(seqs, bs)
    E, scale = ext(), 1.0 / math.sqrt(D)
    out = torch.empty(c["t"], NH * D, dtype=torch.bfloat16, device="cuda")
    paged = lambda: E.attention_fwd_paged(c["q"], c["kc"], c["vc"], c["bt"], c["cu"], c["n"], c["past"], scale, out)   # noqa: E731
    rows = []
    o = 0
    qs = []
    for past, n in seqs:
        qs.append(c["q"][o:o + n])
        o += n
    same = len({(p, n) for p, n in seqs}) == 1
    if same:   # one dense launch over the batch
        Qb, Kb, Vb = torch.stack(qs), torch.stack(c["K"]), torch.stack(c["V"])
        dense = lambda: E.attention_fwd(Qb, Kb, Vb, scale, True)   # noqa: E731
    else:
        dense = lambda: [E.attention_fwd(q[None], k[None], v[None], scale, True) for q, k, v in zip(qs, c["K"], c["V"])]   # noqa: E731
    total = [p + n for p, n in seqs]
    nblk = [(t + bs - 1) // bs for t in total]

    def gather_dense():
        Kg, Vg = [], []
        for i, t in enumerate(total):
            blks = c["bt"][i, :nblk[i]].long()
            Kg.append(c["kc"][blks].permute(0, 2, 1, 3).reshape(nblk[i] * bs, NKV, D)[:t])
            Vg.append(c["vc"][blks].permute(0, 2, 1, 3).reshape(nblk[i] * bs, NKV, D)[:t])
        if same:
            return E.attention_fwd(torch.stack(qs), torch.stack(Kg), torch.stack(Vg), scale, True)
        return [E.attention_fwd(q[None], k[None], v[None], scale, True) for q, k, v in zip(qs, Kg, Vg)]

    fl = causal_flops(seqs)
    res = {"case": label, "block_size": bs, "seqs": len(seqs), "tflop": fl / 1e12}
    impls = [("paged", paged), ("dense", dense), ("gather+dense", gather_dense)]
    if colmask:
        n_all = c["t"]
        qkv_rows = c["q"]
        lens = torch.tensor([n for _, n in seqs], dtype=torch.int64, device="cuda")
        cu_p = torch.zeros(len(seqs) + 1, dtype=torch.int64, device="cuda")
        cu_p[1:] = torch.cumsum(lens, 0)
        k_rows = torch.cat(c["K"])
        v_rows = torch.cat(c["V"])

        def colmask_path():   # the packing the earlier block_attention did for fresh prompts
            pad = (-n_all) % 128
            qp = torch.cat([qkv_rows, qkv_rows.new_zeros(pad, NH, D)]).unsqueeze(0)
            kp = torch.cat([k_rows, k_rows.new_zeros(pad, NKV, D)]).unsqueeze(0)
            vp = torch.cat([v_rows, v_rows.new_zeros(pad, NKV, D)]).unsqueeze(0)
            cm = KAT.colmask_from_cu_seqlens(cu_p, cu_p, n_all + pad)
            return KAT.attention_colmask(qp, kp, vp, cm, causal=True, scale=scale)

        impls.append(("colmask", colmask_path))
    for name, fn in impls:
        ms = timeit(fn)
        res[name + "_ms"] = ms
        res[name + "_tflops"] = fl / ms / 1e9
    return res


def main():
    global ITERS, WARMUP
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="two small cases, few iterations")
    ap.add_argument("--json", default=None, help="also write the results to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_paged_prefill.py needs a CUDA device")
    if a.quick:
        ITERS, WARMUP = 5, 2
    ident = gpu_identity()
    print(json.dumps({"gpu": ident}), flush=True)
    cases = []
    for bs in ((64,) if a.quick else (16, 64)):
        for chunk in ((512,) if a.quick else (512, 2048)):
            for past in ((0, 4096) if a.quick else (0, 4096, 16384)):
                cases.append((f"chunk {chunk} over {past}", [(past, chunk)], bs, False))
        cases.append(("16 x 512 fresh", [(0, 512)] * (4 if a.quick else 16), bs, True))
    results = []
    for label, seqs, bs, cm in cases:
        r = bench_case(label, seqs, bs, cm)
        results.append(r)
        print(json.dumps(r), flush=True)
    print(f"\n{ident['name']}, power limit {ident.get('power_limit')}")
    print(f"{'case':<24}{'bs':>4}{'paged':>16}{'dense':>16}{'gather+dense':>16}{'colmask':>16}   paged/dense")
    for r in results:
        cell = lambda k: f"{r[k + '_ms']:7.3f} {r[k + '_tflops']:6.0f}T" if k + "_ms" in r else ""   # noqa: E731
        print(f"{r['case']:<24}{r['block_size']:>4}{cell('paged'):>16}{cell('dense'):>16}{cell('gather+dense'):>16}{cell('colmask'):>16}"
              f"   {r['dense_ms'] / r['paged_ms']:.2f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"gpu": ident, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
