"""Attention dropout on the sm_90a kernels (csrc/attention_dropout_sm100.cu): three arms on the same bf16 tensors, forward and
forward + backward:

  own p=0.1   the dropout kernels (mask regenerated in the forward and the one-pass backward)
  own p=0     the dropout-free kernels
  sdpa p=0.1  torch SDPA with dropout_p = 0.1 on [B,H,S,D] views (the backend torch picked is read from a profiler run of its own)

Shapes: ERNIE/BERT-base (B 32 x S 512, 12 heads, D 64, non-causal), GPT-350M (B 8 x S 2048, 16 heads, D 64, causal), GPT-1.3B
(B 4 x S 2048, 16 heads, D 128, causal), and the masked case: B 4 x S 4096, 32 / 4 heads, a causal document mask of four 1024-token
documents through flashmask_attention(dropout=0.1), against SDPA with the dense boolean mask (the path it replaces).
e2e: one gpt training step (GPT-350M shapes, 4 layers, B 8 x S 2048) with attention_dropout=0.1, own kernels against
FLAGS_b200_flash_attention=0.

Every shape is warmed up, the arms alternate for --rounds rounds, and each round's time is the median of --reps windows of --iters
calls timed with CUDA events; the table gives the median and (min, max) over the rounds.  The card's name and power limit are read in
the same run.

  python scripts/bench_attention_dropout.py [--parts kernel,masked,e2e] [--rounds 3] [--json FILE]
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
from paddle_b200.nn import functional as PF  # noqa: E402

P = 0.1
SHAPES = [("ernie-base", 32, 512, 12, 12, 64, False), ("gpt-350m", 8, 2048, 16, 16, 64, True), ("gpt-1.3b", 4, 2048, 16, 16, 128, True)]


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


def sdpa_backend(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    for key, label in (("cudnn", "cudnn"), ("flash", "flash"), ("fmha", "mem_efficient"), ("efficient", "mem_efficient")):
        if any(key in n.lower() for n in names):
            return label
    return "math"


def arms_for(q, k, v, causal, mask=None, colmask_fn=None):
    """{arm: (forward fn, forward + backward fn)}; mask: dense bool [S, S] for SDPA."""
    qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
    g = torch.randn_like(q)

    def own(p):
        def fwd():
            with torch.no_grad():
                return colmask_fn(q, k, v, p) if colmask_fn else KAT.attention(q, k, v, None, p, causal)
        def fb():
            qq, kk, vv = (t.detach().requires_grad_(True) for t in (q, k, v))
            o = colmask_fn(qq, kk, vv, p) if colmask_fn else KAT.attention(qq, kk, vv, None, p, causal)
            torch.autograd.backward(o.as_subclass(torch.Tensor), g)
        return fwd, fb

    def sdpa():
        gqa = q.shape[2] != k.shape[2]
        def run(req):
            qq, kk, vv = (t.detach().requires_grad_(req) for t in (qt, kt, vt))
            o = F.scaled_dot_product_attention(qq, kk, vv, attn_mask=mask, dropout_p=P, is_causal=causal and mask is None, enable_gqa=gqa)
            if req:
                torch.autograd.backward(o, g.transpose(1, 2))
        def fwd():
            with torch.no_grad():
                run(False)
        return fwd, lambda: run(True)

    return {"own p=0.1": own(P), "own p=0": own(0.0), "sdpa p=0.1": sdpa()}


def bench_arms(arms, rounds, iters, reps):
    res = {a: {"fwd": [], "fwd+bwd": []} for a in arms}
    for a, (f, fb) in arms.items():   # warm up every arm
        for _ in range(3):
            f(); fb()
    torch.cuda.synchronize()
    for r in range(rounds):
        order = list(arms) if r % 2 == 0 else list(reversed(arms))   # alternate
        for a in order:
            f, fb = arms[a]
            res[a]["fwd"].append(timeit(f, iters, reps))
            res[a]["fwd+bwd"].append(timeit(fb, iters, reps))
    return {a: {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in d.items()} for a, d in res.items()}


def part_kernel(args):
    out = {}
    for name, b, s, h, hk, d, causal in SHAPES:
        gen = torch.Generator(device="cuda").manual_seed(0)
        q, k, v = (torch.randn(b, s, n, d, device="cuda", generator=gen, dtype=torch.bfloat16) for n in (h, hk, hk))
        arms = arms_for(q, k, v, causal)
        out[name] = {"shape": [b, s, h, hk, d, causal], "sdpa_backend": sdpa_backend(arms["sdpa p=0.1"][1]),
                     "arms": bench_arms(arms, args.rounds, args.iters, args.reps)}
        print(name, json.dumps(out[name]), flush=True)
    return out


def part_masked(args):
    b, s, h, hk, d = 4, 4096, 32, 4, 128
    gen = torch.Generator(device="cuda").manual_seed(0)
    q, k, v = (torch.randn(b, s, n, d, device="cuda", generator=gen, dtype=torch.bfloat16) for n in (h, hk, hk))
    doc = torch.arange(s, device="cuda") // 1024
    idx = ((doc + 1) * 1024).to(torch.int32).reshape(1, 1, s, 1).expand(b, 1, s, 1).contiguous()   # rows past a key's document hidden
    dense = (doc.reshape(-1, 1) == doc.reshape(1, -1)) & torch.ones(s, s, dtype=torch.bool, device="cuda").tril()

    def fm(qq, kk, vv, p):
        return PF.flashmask_attention(qq, kk, vv, idx, dropout=p, causal=True)

    arms = arms_for(q, k, v, False, mask=dense, colmask_fn=fm)
    res = {"shape": [b, s, h, hk, d, "causal document mask 4 x 1024"], "sdpa_backend": sdpa_backend(arms["sdpa p=0.1"][1]),
           "arms": bench_arms(arms, args.rounds, args.iters, args.reps)}
    print("masked", json.dumps(res), flush=True)
    return res


def part_e2e(args):
    from paddle_b200.models import GPTForCausalLM, GPTConfig

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    paddle.seed(0)
    cfg = GPTConfig(vocab_size=50304, hidden_size=1024, num_hidden_layers=4, num_attention_heads=16, intermediate_size=4096,
                    max_position_embeddings=2048, attention_dropout=P)
    model = GPTForCausalLM(cfg)
    model.train()
    opt = paddle.optimizer.AdamW(1e-4, parameters=model.parameters(), multi_precision=True)
    ids = torch.randint(0, cfg.vocab_size, (8, 2049), device="cuda")

    def step():
        loss = model(ids[:, :-1], ids[:, 1:])
        loss.backward()
        opt.step()
        opt.clear_grad()

    toks = 8 * 2048
    res = {"own": [], "sdpa": []}
    for arm in res:
        paddle.set_flags({"FLAGS_b200_flash_attention": arm == "own"})
        for _ in range(3):
            step()
    torch.cuda.synchronize()
    for r in range(args.rounds):
        for arm in (("own", "sdpa") if r % 2 == 0 else ("sdpa", "own")):
            paddle.set_flags({"FLAGS_b200_flash_attention": arm == "own"})
            ms = timeit(step, 5, 3)
            res[arm].append(toks / ms * 1e3)
    paddle.set_flags({"FLAGS_b200_flash_attention": True})
    paddle.set_default_dtype("float32")
    out = {a: {"median_tok_s": statistics.median(v), "min": min(v), "max": max(v)} for a, v in res.items()}
    print("e2e", json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernel,masked,e2e")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    result = {"identity": gpu_identity(), "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    parts = args.parts.split(",")
    if "kernel" in parts:
        result["kernel"] = part_kernel(args)
    if "masked" in parts:
        result["masked"] = part_masked(args)
    if "e2e" in parts:
        result["e2e"] = part_e2e(args)
    result["identity_after"] = gpu_identity()
    print(json.dumps(result["identity"]))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
