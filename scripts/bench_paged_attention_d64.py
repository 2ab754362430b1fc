"""Paged attention at head_dim 64 (the 1B-class draft / small-model shape: 32 query / 4 KV heads of 64), bf16, on the sm_90a kernels.

  decode   `decode_attention_paged`, batch 1 / 32 / 128, context 1k / 4k / 16k, block_size 64 and 16.  Beside it the head_dim 128 kernel
           on the same cache bytes per token (32 query / 2 KV heads of 128).  cache GB/s = K and V bytes of every context over the time,
           share = that over the 3.35 TB/s HBM3 data-sheet figure.
  verify   `decode_attention_paged_multi`: rows of 2 .. 5 new tokens over a 4k context, batch 8 / 32 (head_dim 128 beside it where
           n_q * 16 heads fit the 64-row tile).
  prefill  `attention_fwd_paged`: one 2048-token chunk over a cached prefix of 0 / 4096 / 16384 tokens; TFLOP/s counts the causal work
           (4 * D * H per visible query-key pair).  Against torch.nn.functional.scaled_dot_product_attention on the same K / V gathered
           contiguous (bottom-right causal mask; a boolean mask when the prefix is not empty).
  ref      one decode step of batch 8 at context 1k through block_attention, and through `_block_attention_ref` (the path every head_dim
           64 call took before these kernels), host time around device-synchronised calls.
  engine   LLMEngine decode steps with a random-weight Llama-2-7B-shaped target (hidden 4096, 32 / 32 heads of 128, vocab 32000) and a
           TinyLlama-shaped draft (hidden 2048, 32 / 4 heads of 64, intermediate 5632), k = 4 speculative tokens, 8 greedy requests of
           128-token prompts: without a draft, with the draft on the kernels, and with the draft on `_block_attention_ref`.  The layer
           counts are cut to --target-layers / --draft-layers (default 8 of 32 and 6 of 22) to keep the run short.  Each step is timed
           on the host between device synchronizes; median and spread (min, max) of the round medians.  With random weights the draft's
           proposals are almost never accepted, so a speculative step yields about one token per sequence.

Kernel times are medians of CUDA-event times (bench_paged_prefill.timeit).  The card's name and power limit are read in the same run.

  python scripts/bench_paged_attention_d64.py [--parts decode,verify,prefill,ref,engine] [--json FILE]
"""
import argparse
import json
import math
import os
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench_paged_prefill as BP  # noqa: E402
import paddle_b200 as paddle  # noqa: E402
from paddle_b200._build import ext  # noqa: E402
from paddle_b200.incubate.nn import paged_attention as PA  # noqa: E402

NH = 32
HBM = 3.35e12
SHAPES = {64: 4, 128: 2}          # head_dim -> KV heads: the same cache bytes per token


def i32(v):
    return torch.tensor(v, dtype=torch.int32, device="cuda")


def paged(batch, ctx, nkv, d, bs, g):
    nblk = (ctx + bs - 1) // bs
    bt = torch.randperm(batch * nblk, device="cuda", generator=g).to(torch.int32).reshape(batch, nblk).contiguous()
    kc = (torch.randn(batch * nblk, nkv, bs, d, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    return bt, kc, torch.randn_like(kc)


def rate(nbytes, ms):
    return {"us": round(ms * 1e3, 1), "cache_GBps": round(nbytes / ms / 1e6, 1), "share_of_hbm": round(nbytes / ms / 1e-3 / HBM, 3)}


def bench_decode():
    rows = []
    g = torch.Generator(device="cuda").manual_seed(0)
    for bs in (64, 16):
        for batch in (1, 32, 128):
            for ctx in (1024, 4096, 16384):
                row = {"part": "decode", "block_size": bs, "batch": batch, "context": ctx}
                for d, nkv in SHAPES.items():
                    bt, kc, vc = paged(batch, ctx, nkv, d, bs, g)
                    q = torch.randn(batch, NH, d, device="cuda", generator=g).to(torch.bfloat16)
                    lens = i32([ctx] * batch)
                    ms = BP.timeit(lambda: ext().decode_attention_paged(q, kc, vc, lens, bt, 1 / math.sqrt(d)))
                    row[f"d{d}"] = rate(2 * batch * ctx * nkv * d * 2, ms)
                    del kc, vc
                print(json.dumps(row), flush=True)
                rows.append(row)
    return rows


def bench_verify():
    rows = []
    g = torch.Generator(device="cuda").manual_seed(1)
    ctx, bs = 4096, 64
    for batch in (8, 32):
        for nq in (2, 3, 4, 5):
            row = {"part": "verify", "block_size": bs, "batch": batch, "context": ctx, "n_q": nq}
            for d, nkv in SHAPES.items():
                if nq * (NH // nkv) > 64:
                    continue
                bt, kc, vc = paged(batch, ctx + nq, nkv, d, bs, g)
                q = torch.randn(batch * nq, NH, d, device="cuda", generator=g).to(torch.bfloat16)
                out = torch.empty(batch * nq, NH * d, device="cuda", dtype=torch.bfloat16)
                cu, n, past = i32([b * nq for b in range(batch)]), i32([nq] * batch), i32([ctx] * batch)
                ms = BP.timeit(lambda: ext().decode_attention_paged_multi(q, kc, vc, bt, cu, n, past, 1 / math.sqrt(d), out))
                row[f"d{d}"] = rate(2 * batch * (ctx + nq) * nkv * d * 2, ms)
                del kc, vc
            print(json.dumps(row), flush=True)
            rows.append(row)
    return rows


def bench_prefill():
    rows = []
    g = torch.Generator(device="cuda").manual_seed(2)
    d, nkv, chunk = 64, SHAPES[64], 2048
    for bs in (64, 16):
        for past in (0, 4096, 16384):
            bt, kc, vc = paged(1, past + chunk, nkv, d, bs, g)
            q = torch.randn(chunk, NH, d, device="cuda", generator=g).to(torch.bfloat16)
            out = torch.empty(chunk, NH * d, device="cuda", dtype=torch.bfloat16)
            ms = BP.timeit(lambda: ext().attention_fwd_paged(q, kc, vc, bt, i32([0]), i32([chunk]), i32([past]), 1 / math.sqrt(d), out))
            flops = 4.0 * d * NH * (chunk * past + chunk * (chunk + 1) // 2)
            # the same K / V gathered contiguous for SDPA: [1, H, S, D], KV heads repeated
            k = kc[bt[0].long()].permute(1, 0, 2, 3).reshape(nkv, -1, d)[:, :past + chunk].repeat_interleave(NH // nkv, 0)[None]
            v = vc[bt[0].long()].permute(1, 0, 2, 3).reshape(nkv, -1, d)[:, :past + chunk].repeat_interleave(NH // nkv, 0)[None]
            qs = q.permute(1, 0, 2)[None].contiguous()
            if past == 0:
                sdpa = lambda: torch.nn.functional.scaled_dot_product_attention(qs, k, v, is_causal=True)   # noqa: E731
            else:
                mask = torch.arange(past + chunk, device="cuda")[None] <= (past + torch.arange(chunk, device="cuda"))[:, None]
                sdpa = lambda: torch.nn.functional.scaled_dot_product_attention(qs, k, v, attn_mask=mask)   # noqa: E731
            ref = sdpa()[0].permute(1, 0, 2).reshape(chunk, NH * d)
            err = ((out.float() - ref.float()).norm() / ref.float().norm()).item()
            ms_sdpa = BP.timeit(sdpa)
            row = {"part": "prefill", "block_size": bs, "chunk": chunk, "past": past, "ms": round(ms, 3), "TFLOPs": round(flops / ms / 1e9, 1),
                   "sdpa_ms": round(ms_sdpa, 3), "sdpa_TFLOPs": round(flops / ms_sdpa / 1e9, 1), "speedup_vs_sdpa": round(ms_sdpa / ms, 2),
                   "rel_err_vs_sdpa": round(err, 5)}
            print(json.dumps(row), flush=True)
            rows.append(row)
            del kc, vc, k, v
    return rows


def host_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts)


def bench_ref():
    g = torch.Generator(device="cuda").manual_seed(3)
    d, nkv, bs, batch, ctx = 64, SHAPES[64], 64, 8, 1024
    bt, kc, vc = paged(batch, ctx, nkv, d, bs, g)
    qkv = torch.randn(batch, (NH + 2 * nkv) * d, device="cuda", generator=g).to(torch.bfloat16)
    args = (i32([0] * batch), i32([ctx - 1] * batch), i32([1] * batch), i32(list(range(batch + 1))), bt, bs)
    kern = host_ms(lambda: PA.block_attention(qkv, kc, vc, *args), 50)
    ref = host_ms(lambda: PA._block_attention_ref(qkv, kc, vc, *args), 5)
    row = {"part": "ref", "batch": batch, "context": ctx, "block_size": bs, "kernel_ms": round(kern, 3), "reference_ms": round(ref, 2),
           "reference_over_kernel": round(ref / kern, 1)}
    print(json.dumps(row), flush=True)
    return [row]


def bench_engine(target_layers, draft_layers, steps, rounds):
    from paddle_b200 import models

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        target = models.LlamaForCausalLM(models.LlamaConfig(vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_attention_heads=32,
                                                            num_key_value_heads=32, num_hidden_layers=target_layers, max_position_embeddings=4096))
        draft = models.LlamaForCausalLM(models.LlamaConfig(vocab_size=32000, hidden_size=2048, intermediate_size=5632, num_attention_heads=32,
                                                           num_key_value_heads=4, num_hidden_layers=draft_layers, max_position_embeddings=4096))
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, 32000, (128,), generator=g).tolist() for _ in range(8)]
    kernels_ok = PA._paged_kernels_ok
    rows = []
    for label, kw, ref in (("no_draft", {}, False), ("draft_kernels", dict(draft_model=draft, num_speculative_tokens=4), False),
                           ("draft_reference", dict(draft_model=draft, num_speculative_tokens=4), True)):
        if ref:   # the head_dim 64 draft on the reference path, as before these kernels
            PA._paged_kernels_ok = lambda qkv, kc, d, *a, **k: d != 64 and kernels_ok(qkv, kc, d, *a, **k)
        try:
            eng = models.LLMEngine(target, num_blocks=8 * ((128 + 5 * (steps * rounds + 8)) // 16 + 2), block_size=16, max_running=8, **kw)
            for p in prompts:
                eng.add_request(p, 5 * (steps * rounds + 8))
            eng.step()                                               # every prompt prefills in this step
            for _ in range(3):
                eng.step()
            meds, toks = [], []
            for _ in range(rounds):
                ts = []
                for _ in range(steps):
                    before = sum(len(s.generated) for s in eng.running)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    eng.step()
                    torch.cuda.synchronize()
                    ts.append((time.perf_counter() - t0) * 1e3)
                    toks.append(sum(len(s.generated) for s in eng.running) - before)
                meds.append(statistics.median(ts))
        finally:
            PA._paged_kernels_ok = kernels_ok
        row = {"part": "engine", "arm": label, "target_layers": f"{target_layers} of 32", "draft_layers": f"{draft_layers} of 22", "running": 8,
               "step_ms_median": round(statistics.median(meds), 1), "step_ms_min": round(min(meds), 1), "step_ms_max": round(max(meds), 1),
               "tokens_per_step": round(statistics.mean(toks), 2), "rounds": rounds, "steps_per_round": steps}
        print(json.dumps(row), flush=True)
        rows.append(row)
        del eng
        torch.cuda.empty_cache()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="decode,verify,prefill,ref,engine")
    ap.add_argument("--target-layers", type=int, default=8)
    ap.add_argument("--draft-layers", type=int, default=6)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_paged_attention_d64.py measures the GPU; there is nothing to measure without one"
    ident = BP.gpu_identity()
    print(json.dumps({"gpu": ident}), flush=True)
    parts = a.parts.split(",")
    rows = []
    for name, fn in (("decode", bench_decode), ("verify", bench_verify), ("prefill", bench_prefill), ("ref", bench_ref)):
        if name in parts:
            rows += fn()
    if "engine" in parts:
        rows += bench_engine(a.target_layers, a.draft_layers, a.steps, a.rounds)
    print(f"\n{ident['name']}, power limit {ident.get('power_limit')}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"gpu": ident, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
