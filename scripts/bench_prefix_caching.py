"""Prefix caching: the shared-prefix decode kernel, and LLMEngine with and without enable_prefix_caching.

Kernel part: one group of B single-token decode rows whose first `prefix` cached tokens are the same blocks, plus `suffix` = 64 own keys
each (the new token included), block_size 64.  Heads 32 / 8 and 32 / 32 of 128, bf16 queries, bf16 and int8 caches, B 2 / 4 / 16 / 64,
prefix 512 / 1k / 4k / 16k.  On the same rows it times
  shared  `decode_attention_paged_shared` (csrc/decode_attention.cu), one call for the group (the host builds its task list in the call)
  decode  `decode_attention_paged`, which reads the prefix once per sequence
Each time is the median over 10 windows of 20 back-to-back calls (after 3 warm-up calls), per call, from CUDA events.  "GB/s" is the
unique cache bytes - the K and V rows of the prefix once plus every member's suffix - over that time.

Engine part: 32 requests sharing a 2,048-token system prompt plus 32 unique tokens each, 64 new tokens each, all added at once, on a
random-weight Llama (head_dim 128, bf16, block_size 64), with prefix caching on and off: wall time to completion, time until every request
has its first token, and prefill_tokens; with caching on, also with every decode row kept on `decode_attention_paged`.  The card's name and power limit are printed with the results.

  python scripts/bench_prefix_caching.py [--quick] [--skip-kernels] [--engine-repeats N] [--json FILE]
"""
import argparse
import json
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_paged_prefill import gpu_identity  # noqa: E402
from paddle_b200._build import ext  # noqa: E402

NH, D, BS, SUFFIX = 32, 128, 64, 64
WINDOWS, CALLS, WARMUP = 10, 20, 3


def timeit(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(WINDOWS):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(CALLS):
            fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) * 1e3 / CALLS)
    ts.sort()
    return ts[len(ts) // 2]


def kernel_case(nkv, kind, b, prefix, g):
    npre, nown = prefix // BS, (SUFFIX + BS - 1) // BS
    nblocks = npre + b * nown
    perm = torch.randperm(nblocks, device="cuda", generator=g).to(torch.int32)
    bt = torch.empty(b, npre + nown, dtype=torch.int32, device="cuda")
    bt[:, :npre] = perm[:npre]
    bt[:, npre:] = perm[npre:].reshape(b, nown)
    shape = (nblocks, nkv, BS, D)
    if kind == "int8":
        kc, vc = (torch.randint(-127, 128, shape, generator=g, device="cuda", dtype=torch.int8) for _ in range(2))
        dq = dict(k_dequant_scales=torch.full((nkv,), 0.01, device="cuda"), v_dequant_scales=torch.full((nkv,), 0.01, device="cuda"))
    else:
        kc, vc = ((torch.randn(shape, generator=g, device="cuda") * 0.5).to(torch.bfloat16) for _ in range(2))
        dq = {}
    q = (torch.randn(b, NH, D, generator=g, device="cuda") * 0.5).to(torch.bfloat16)
    lens = torch.full((b,), prefix + SUFFIX, dtype=torch.int32, device="cuda")
    cu_q = torch.arange(b, dtype=torch.int32, device="cuda")
    groups = (torch.tensor([0, b], dtype=torch.int32), torch.arange(b, dtype=torch.int32), torch.tensor([prefix], dtype=torch.int32))
    scale = 1.0 / math.sqrt(D)
    out = torch.empty(b, NH * D, dtype=torch.bfloat16, device="cuda")
    X = ext()

    def shared():
        X.decode_attention_paged_shared(q, kc, vc, bt, cu_q, lens, *groups, scale, out, **dq)

    def decode():
        return X.decode_attention_paged(q, kc, vc, lens, bt, scale, **dq)

    shared()
    ref = decode().reshape(b, NH * D).float()
    err = ((out.float() - ref).norm() / ref.norm()).item()
    t_sh, t_dec = timeit(shared), timeit(decode)
    elem = 1 if kind == "int8" else 2
    uniq = 2 * (prefix + b * SUFFIX) * nkv * D * elem
    return {"heads": f"{NH}/{nkv}", "cache": kind, "group": b, "prefix": prefix, "shared_us": t_sh, "decode_us": t_dec,
            "shared_GBps": uniq / t_sh / 1e3, "decode_GBps": uniq / t_dec / 1e3, "speedup": t_dec / t_sh, "rel_err": err}


def engine_case(caching, quick, grouping=True):
    import paddle_b200 as paddle
    from paddle_b200 import models
    from paddle_b200.incubate.nn import paged_attention as PA

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.llama_tiny(hidden_size=2048, intermediate_size=5632, num_attention_heads=16, num_key_value_heads=4,
                                num_hidden_layers=2 if quick else 8, vocab_size=32000, max_position_embeddings=4096)
        m = models.LlamaForCausalLM(cfg)
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    g = torch.Generator().manual_seed(0)
    n_req, sys_len, uniq, new = (8, 512, 32, 8) if quick else (32, 2048, 32, 64)
    system = torch.randint(1, cfg.vocab_size, (sys_len,), generator=g).tolist()
    prompts = [system + torch.randint(1, cfg.vocab_size, (uniq,), generator=g).tolist() for _ in range(n_req)]
    blocks = n_req * ((sys_len + uniq + new + BS - 1) // BS) + 8
    res = {}
    saved = PA.SHARED_PREFIX_MIN_GROUP, PA.SHARED_PREFIX_LARGE_GROUP
    if not grouping:                                   # caching on, every decode row on decode_attention_paged
        PA.SHARED_PREFIX_MIN_GROUP = PA.SHARED_PREFIX_LARGE_GROUP = 1 << 30
    for rep in ("warm-up", "timed"):
        eng = models.LLMEngine(m, num_blocks=blocks, block_size=BS, max_running=n_req, enable_prefix_caching=caching)
        for p in prompts:
            eng.add_request(p, new)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        first = None
        while eng.has_unfinished():
            eng.step()
            if first is None and all(len(s.generated) > 0 for s in eng.running) and not eng.waiting:
                torch.cuda.synchronize()
                first = time.perf_counter() - t0
        torch.cuda.synchronize()
        res = {"prefix_caching": caching, "requests": n_req, "wall_s": time.perf_counter() - t0, "all_first_token_s": first,
               "prefill_tokens": eng.stats["prefill_tokens"], "prefix_hit_tokens": eng.stats.get("prefix_hit_tokens", 0),
               "steps": eng.stats["steps"], "shared_decode": caching and grouping}
    PA.SHARED_PREFIX_MIN_GROUP, PA.SHARED_PREFIX_LARGE_GROUP = saved
    return res


def main():
    global WINDOWS, CALLS
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--json")
    ap.add_argument("--engine-repeats", type=int, default=1, help="timed engine runs per setting, alternating off / on")
    ap.add_argument("--skip-kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_prefix_caching.py needs a GPU")
    if a.quick:
        WINDOWS, CALLS = 3, 5
    ident = gpu_identity()
    print(json.dumps(ident))
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    print("| heads | cache | group | prefix | shared µs | decode µs | shared GB/s | decode GB/s | decode / shared |")
    print("|---|---|---:|---:|---:|---:|---:|---:|---:|")
    for nkv in (() if a.skip_kernels else (8, 32)):
        for kind in ("bf16", "int8"):
            for b in ((4, 16) if a.quick else (2, 4, 16, 64)):
                for prefix in ((1024,) if a.quick else (512, 1024, 4096, 16384)):
                    r = kernel_case(nkv, kind, b, prefix, g)
                    assert r["rel_err"] < 2e-2, r
                    rows.append(r)
                    print(f"| {r['heads']} | {kind} | {b} | {prefix} | {r['shared_us']:.1f} | {r['decode_us']:.1f} | {r['shared_GBps']:.0f} | "
                          f"{r['decode_GBps']:.0f} | {r['speedup']:.2f} |", flush=True)
    eng = [engine_case(c, a.quick, grp) for _ in range(a.engine_repeats) for c, grp in ((False, True), (True, True), (True, False))]
    print("| prefix caching | shared-prefix decode | wall s | all first tokens s | prefill_tokens | prefix_hit_tokens | steps |")
    print("|---|---|---:|---:|---:|---:|---:|")
    for r in eng:
        print(f"| {'on' if r['prefix_caching'] else 'off'} | {'yes' if r['shared_decode'] else 'no'} | {r['wall_s']:.2f} | {r['all_first_token_s']:.2f} | {r['prefill_tokens']} | "
              f"{r['prefix_hit_tokens']} | {r['steps']} |")
    print(json.dumps(ident))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({"gpu": ident, "kernel": rows, "engine": eng}, f, indent=1)


if __name__ == "__main__":
    main()
