"""Column-masked attention that skips the tiles the mask hides (csrc/attention_flashmask_sm100.cu), bf16, forward and forward + backward,
four arms on the same tensors:

  skip      the tile-skipping kernels (the default)
  masked    the kernels that test every element of every tile up to the causal limit (B200_ATTN_MASK_SKIP=0, switched in-process)
  per-doc   the dense causal kernels called once per document (the work-optimal bound; document masks only)
  sdpa      torch SDPA with the dense boolean mask

Shapes: B 4 x S 4096, 32 / 4 heads, D 128 with causal documents 4 x 1024, 16 x 256 and a seeded mix of lengths; TinyLlama's B 8 x S 2048,
32 / 4, D 64 with 8 documents; Mistral's 4096-token window at B 1 x S 16384, 32 / 8, D 128; and one general 4-bound flashmask (both
intervals, not causal) at B 4 x S 4096.  Beside each time: the fraction of the forward's score tiles the skipping kernels compute,
from kernels.attention.colmask_tile_classes (shapes only), against the tiles the masked kernels walk.
e2e: tinyllama_1b() training steps (AdamW) at B 4 x S 2048 with 4 documents per row, in tokens/s: skip, masked, and no document mask.

Every shape is warmed up, the arms alternate for --rounds rounds, and each round's time is the median of --reps windows of --iters
calls timed with CUDA events; the tables give the median and (min, max) over the rounds.  The card's name and power limit are read in
the same run.

  python scripts/bench_flashmask.py [--parts kernel,e2e] [--rounds 3] [--json FILE]
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
from paddle_b200.kernels import attention as KAT  # noqa: E402

INT_MAX = 2 ** 31 - 1


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    name, power, clock = (x.strip() for x in r.stdout.strip().split(",")[:3])
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def timeit(fn, iters, reps):
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


def doc_lengths(kind, s, seed=0):
    if kind.startswith("docs"):
        n = int(kind.split(":")[1])
        return [s // n] * n
    g = torch.Generator().manual_seed(seed)   # "mix": lengths 64 .. 2048 until the row is full
    lens = []
    while sum(lens) < s:
        lens.append(min(int(torch.randint(64, 2049, (1,), generator=g)), s - sum(lens)))
    return lens


def doc_colmask(b, lens, device):
    ends = torch.cat([torch.full((n,), e, dtype=torch.int32) for n, e in zip(lens, torch.tensor(lens).cumsum(0).tolist())])
    return KAT.colmask_from_startend(ends.reshape(1, 1, -1, 1).expand(b, 1, -1, 1).to(device), True, ends.numel())


def four_bound_colmask(b, s, device):
    """Both intervals, block-structured: key j (block of 512) is seen by the rows of a band around it, [j0 - 1024, j0 + 1024)."""
    j0 = torch.arange(s, device=device) // 512 * 512
    lts, lte = (j0 + 1024).clamp(max=s), torch.full_like(j0, INT_MAX)
    uts, ute = torch.zeros_like(j0), (j0 - 1024).clamp(min=0)
    return torch.stack([lts, lte, uts, ute], -1).int().reshape(1, 1, s, 4).expand(b, 1, s, 4).contiguous()


def tile_fraction(cm, s, causal):
    new = int((KAT.colmask_tile_classes(cm[:1], s, s, 128, 128, causal) != 0).sum())
    walk = int((KAT.colmask_tile_classes(torch.zeros_like(cm[:1]), s, s, 128, 128, causal) != 0).sum())
    return {"computed_tiles": new, "walked_by_masked": walk, "fraction": new / walk}


def arms_for(q, k, v, cm, causal, lens):
    g = torch.randn_like(q)
    s = q.shape[1]

    def own(skip):
        def call(qq, kk, vv):
            KAT._mask_skip[0] = skip
            try:
                return KAT.attention_colmask(qq, kk, vv, cm, causal=causal)
            finally:
                KAT._mask_skip[0] = True
        def fwd():
            with torch.no_grad():
                call(q, k, v)
        def fb():
            qq, kk, vv = (t.detach().requires_grad_(True) for t in (q, k, v))
            torch.autograd.backward(call(qq, kk, vv).as_subclass(torch.Tensor), g)
        return fwd, fb

    def per_doc():
        offs = [0] + torch.tensor(lens).cumsum(0).tolist()
        def run(req):
            for a, e in zip(offs[:-1], offs[1:]):
                qq, kk, vv = (t[:, a:e].detach().requires_grad_(req) for t in (q, k, v))
                o = KAT.attention(qq, kk, vv, None, 0.0, True)
                if req:
                    torch.autograd.backward(o.as_subclass(torch.Tensor), g[:, a:e])
        def fwd():
            with torch.no_grad():
                run(False)
        return fwd, lambda: run(True)

    def sdpa():
        vis = KAT.colmask_to_dense(cm, s)
        if causal:
            vis = vis & torch.ones(s, s, dtype=torch.bool, device=q.device).tril()
        qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
        def run(req):
            qq, kk, vv = (t.detach().requires_grad_(req) for t in (qt, kt, vt))
            o = F.scaled_dot_product_attention(qq, kk, vv, attn_mask=vis, enable_gqa=q.shape[2] != k.shape[2])
            if req:
                torch.autograd.backward(o, g.transpose(1, 2))
        def fwd():
            with torch.no_grad():
                run(False)
        return fwd, lambda: run(True)

    arms = {"skip": own(True), "masked": own(False)}
    if lens is not None:
        arms["per-doc"] = per_doc()
    arms["sdpa"] = sdpa()
    return arms


def bench_arms(arms, rounds, iters, reps):
    res = {a: {"fwd": [], "fwd+bwd": []} for a in arms}
    errors = {}
    for a in list(arms):   # warm up every arm
        try:
            for _ in range(2):
                arms[a][0](); arms[a][1]()
            torch.cuda.synchronize()
        except torch.OutOfMemoryError as e:   # SDPA's dense mask at the longest shape
            errors[a] = str(e).split("\n")[0]
            del arms[a], res[a]
            torch.cuda.empty_cache()
    for r in range(rounds):
        for a in (list(arms) if r % 2 == 0 else list(reversed(arms))):   # alternate
            f, fb = arms[a]
            res[a]["fwd"].append(timeit(f, iters, reps))
            res[a]["fwd+bwd"].append(timeit(fb, iters, reps))
    out = {a: {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in d.items()} for a, d in res.items()}
    out.update({a: {"error": e} for a, e in errors.items()})
    return out


SHAPES = [  # name, b, s, h, hk, d, mask
    ("docs 4x1024", 4, 4096, 32, 4, 128, "docs:4"),
    ("docs 16x256", 4, 4096, 32, 4, 128, "docs:16"),
    ("docs mix", 4, 4096, 32, 4, 128, "mix"),
    ("tinyllama 8 docs", 8, 2048, 32, 4, 64, "docs:8"),
    ("mistral window 4096", 1, 16384, 32, 8, 128, "window"),
    ("4-bound flashmask", 4, 4096, 32, 4, 128, "4-bound"),
]


def part_kernel(args):
    out = {}
    for name, b, s, h, hk, d, kind in SHAPES:
        gen = torch.Generator(device="cuda").manual_seed(0)
        q, k, v = (torch.randn(b, s, n, d, device="cuda", generator=gen, dtype=torch.bfloat16) for n in (h, hk, hk))
        lens, causal = None, True
        if kind == "window":
            cm = KAT.colmask_from_window(s, s, 4095, 0, True, "cuda").expand(b, 1, s, 4).contiguous()
        elif kind == "4-bound":
            cm, causal = four_bound_colmask(b, s, "cuda"), False
        else:
            lens = doc_lengths(kind, s)
            cm = doc_colmask(b, lens, "cuda")
        res = {"shape": [b, s, h, hk, d, kind], "causal": causal, "tiles": tile_fraction(cm, s, causal),
               "arms": bench_arms(arms_for(q, k, v, cm, causal, lens), args.rounds, args.iters, args.reps)}
        if lens is not None:
            res["documents"] = lens
        out[name] = res
        print(name, json.dumps(res), flush=True)
        del q, k, v
        torch.cuda.empty_cache()
    return out


def part_e2e(args):
    from paddle_b200.models import LlamaForCausalLM, tinyllama_1b

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    paddle.seed(0)
    cfg = tinyllama_1b()
    model = LlamaForCausalLM(cfg)
    model.train()
    opt = paddle.optimizer.AdamW(1e-4, parameters=model.parameters(), multi_precision=True)
    b, s = 4, 2048
    ids = torch.randint(0, cfg.vocab_size, (b, s + 1), device="cuda")
    lens = [512] * 4
    ends = torch.cat([torch.full((n,), e) for n, e in zip(lens, torch.tensor(lens).cumsum(0).tolist())])
    se = ends.reshape(1, 1, s, 1).expand(b, 1, s, 1).int().cuda().as_subclass(paddle.Tensor)
    pos = torch.cat([torch.arange(n) for n in lens]).reshape(1, s).expand(b, s).cuda().as_subclass(paddle.Tensor)
    x, y = ids[:, :-1].as_subclass(paddle.Tensor), ids[:, 1:].as_subclass(paddle.Tensor)

    def step_for(arm):
        def step():
            KAT._mask_skip[0] = arm != "masked"
            loss = model(x, y, pos, se) if arm != "no mask" else model(x, y)
            loss.backward()
            opt.step()
            opt.clear_grad()
            KAT._mask_skip[0] = True
        return step

    res = {"skip": [], "masked": [], "no mask": []}
    for arm in res:
        for _ in range(3):
            step_for(arm)()
    torch.cuda.synchronize()
    for r in range(args.rounds):
        for arm in (list(res) if r % 2 == 0 else list(reversed(res))):
            ms = timeit(step_for(arm), 5, 3)
            res[arm].append(b * s / ms * 1e3)
    paddle.set_default_dtype("float32")
    out = {a: {"median_tok_s": statistics.median(v), "min": min(v), "max": max(v)} for a, v in res.items()}
    print("e2e", json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernel,e2e")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_flashmask.py measures on the GPU"
    result = {"identity": gpu_identity(), "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    parts = args.parts.split(",")
    if "kernel" in parts:
        result["kernel"] = part_kernel(args)
    if "e2e" in parts:
        result["e2e"] = part_e2e(args)
    result["identity_after"] = gpu_identity()
    print(json.dumps(result["identity"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
