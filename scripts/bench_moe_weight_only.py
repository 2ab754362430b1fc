"""Weight-only int8 / int4 MoE experts on the GPU: the whole expert FFN (routing plan, scatter, two expert GEMMs, SwiGLU, combine) of one
MoE layer, timed per route over routed slot counts from decode to prefill sizes.

  shapes    mixtral   Mixtral-8x7B's MoE layer: d 4096, f 14336, 8 experts, top-2.
            many      a many-expert layer: d 2048, f 1408, 64 experts, top-6.
  arms      bf16      `kernels.moe.expert_ffn_grouped` on 16-bit weights.
            insm      int8 / int4 x per-channel / g128 on the in-SM route (`expert_ffn_in_sm`, at every slot count).
            deq       int8 per-channel and int4-g128 on the dequantise route (`expert_ffn_dequantized`).
  timing    `calls` expert FFN calls captured into one CUDA graph (the in-SM route has no host synchronisation), each call with its own
            random routing so that a replay does not find its experts' weights in the 50 MB L2; the median of 5 replays per call.
  bytes     the weight (and scale) bytes of the experts the routings select, averaged over the calls; "of_peak" divides bytes / time by
            the data sheet's 3.35 TB/s.  Weight-stack sizes are computed from the shapes, not measured.

The card's name and power limit are read in the same run and printed with the numbers.  The crossover per format is the smallest slot
count at which the dequantise route is at least as fast as the in-SM route.

  python scripts/bench_moe_weight_only.py [--shapes mixtral,many] [--tokens 1,4,16,...] [--calls N] [--json FILE]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_paged_prefill import gpu_identity  # noqa: E402
import paddle_b200 as paddle  # noqa: E402
from paddle_b200.kernels import moe as KM  # noqa: E402
from paddle_b200.nn import quant as Q  # noqa: E402

HBM = 3.35e12
SHAPES = {"mixtral": dict(d=4096, f=14336, E=8, topk=2), "many": dict(d=2048, f=1408, E=64, topk=6)}
FORMATS = [("int8", -1), ("int8", 128), ("int4", -1), ("int4", 128)]
DEQ_FORMATS = [("int8", -1), ("int4", 128)]


def graph_time(fns, replays=5):
    """Device time per call: the calls `fns` captured into one CUDA graph, replayed; median replay over `replays`."""
    for fn in fns[:2]:
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        fns[0]()
        st.synchronize()
        with torch.cuda.graph(g, stream=st):
            for fn in fns:
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
        ts.append(a.elapsed_time(b) / len(fns))
    g.reset()
    return statistics.median(ts)


def quantize_stack(w, wdt, gs):
    """[E, K, N] 16-bit -> (q int8 [E, N, K] (int4 [E, N, K/2]), fp32 scales [E, N] or [E, K/gs, N])."""
    qs = [Q.weight_quantize(w[e].as_subclass(paddle.Tensor), algo=f"weight_only_{wdt}", group_size=gs) for e in range(w.shape[0])]
    q = torch.stack([q.as_subclass(torch.Tensor) for q, _ in qs]).contiguous()
    s = torch.stack([s.as_subclass(torch.Tensor).float() for _, s in qs]).contiguous()
    return q, s


def expert_bytes(d, f, wdt, gs):
    """Bytes one expert's two weights (and their scales) occupy."""
    n_w = d * 2 * f + f * d
    if wdt == "bf16":
        return 2 * n_w
    wb = n_w // 2 if wdt == "int4" else n_w
    sc = (2 * f + d) * 4 if gs < 0 else (d // gs * 2 * f + f // gs * d) * 4
    return wb + sc


def run_shape(name, cfg, tokens, calls):
    d, f, E, topk = cfg["d"], cfg["f"], cfg["E"], cfg["topk"]
    gen = torch.Generator(device="cuda").manual_seed(0)
    w1 = (torch.randn(E, d, 2 * f, device="cuda", generator=gen) * 0.02).to(torch.bfloat16)
    w2 = (torch.randn(E, f, d, device="cuda", generator=gen) * 0.02).to(torch.bfloat16)
    quant = {fmt: (quantize_stack(w1, *fmt), quantize_stack(w2, *fmt)) for fmt in FORMATS}
    rows = []
    for T in tokens:
        x = (torch.randn(T, d, device="cuda", generator=gen) * 0.5).to(torch.bfloat16)
        routes = []
        for _ in range(calls):
            val, idx = torch.softmax(torch.randn(T, E, device="cuda", generator=gen), -1).topk(topk, -1)
            routes.append((idx, (val / val.sum(-1, keepdim=True)).float()))
        active = statistics.mean(len(set(idx.reshape(-1).tolist())) for idx, _ in routes)
        S = T * topk
        row = dict(shape=name, T=T, slots=S, active_experts=active)

        def record(arm, fmt, fns):
            us = graph_time(fns) * 1e3
            nbytes = active * expert_bytes(d, f, *fmt)
            row[arm] = dict(us=round(us, 1), active_weight_MB=round(nbytes / 1e6, 1), of_peak=round(nbytes / (us * 1e-6) / HBM, 3))

        with torch.no_grad():
            record("bf16", ("bf16", -1), [lambda r=r: KM.expert_ffn_grouped(x, r[0], r[1], w1, w2) for r in routes])
            for wdt, gs in FORMATS:
                (q1, s1), (q2, s2) = quant[(wdt, gs)]
                tag = f"{wdt}_{'pc' if gs < 0 else 'g' + str(gs)}"
                record("insm_" + tag, (wdt, gs), [lambda r=r, a=(q1, s1, q2, s2, wdt == "int4", gs): KM.expert_ffn_in_sm(x, r[0], r[1], *a)
                                                  for r in routes])
                if (wdt, gs) in DEQ_FORMATS:
                    record("deq_" + tag, (wdt, gs), [lambda r=r, a=(q1, s1, q2, s2, wdt == "int4", gs): KM.expert_ffn_dequantized(x, r[0], r[1], *a)
                                                     for r in routes[:4]])
        rows.append(row)
        print(json.dumps(row), flush=True)
    return rows


def crossovers(rows):
    out = {}
    for wdt, gs in DEQ_FORMATS:
        tag = f"{wdt}_{'pc' if gs < 0 else 'g' + str(gs)}"
        for shape in sorted({r["shape"] for r in rows}):
            first = next((r["slots"] for r in rows if r["shape"] == shape and r["deq_" + tag]["us"] <= r["insm_" + tag]["us"]), None)
            out[f"{shape}_{tag}"] = first
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="mixtral,many")
    ap.add_argument("--tokens", default="1,4,16,32,64,128,512,2048")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_moe_weight_only needs a GPU")
    ident = gpu_identity()
    print(json.dumps(ident), flush=True)
    for name in a.shapes.split(","):
        cfg = SHAPES[name]
        d, f, E = cfg["d"], cfg["f"], cfg["E"]
        sizes = {fmt: E * expert_bytes(d, f, *fmt) / 1e9 for fmt in [("bf16", -1)] + FORMATS}
        print(json.dumps({"shape": name, "computed_expert_stack_GB": {f"{w}_{g}": round(v, 2) for (w, g), v in sizes.items()}}), flush=True)
    tokens = [int(t) for t in a.tokens.split(",")]
    rows = [r for name in a.shapes.split(",") for r in run_shape(name, SHAPES[name], tokens, a.calls)]
    cross = crossovers(rows)
    print(json.dumps({"crossover_slots": cross, "WO_MOE_MAX_SLOTS": KM.WO_MOE_MAX_SLOTS}), flush=True)
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(dict(gpu=ident, rows=rows, crossover_slots=cross), fh, indent=1)


if __name__ == "__main__":
    main()
