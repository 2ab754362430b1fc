"""Sliding-window attention without a GPU: block_attention's reference under a window against dense masked attention, the argument checks,
LlamaForCausalLM with a window against an explicit-mask forward, LLMEngine's block release against generate(), and the windowed kernels
in the built attention objects (no local memory, pipelined wgmma)."""
import math
import os
import re
import shutil
import subprocess

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models
from paddle_b200.incubate.nn.paged_attention import _block_attention_ref, block_attention

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WINDOW_OBJS = [os.path.join(ROOT, "paddle_b200", "_build_cache", f) for f in ("attention_sm100.cuda.o", "decode_attention.cuda.o")]


def _dense(q, k, v, window):
    """q [n, H, D] at positions past .. past + n - 1, k / v [past + n, Hkv, D]: causal sliding-window attention in float64."""
    n, h, d = q.shape
    total, hkv = k.shape[0], k.shape[1]
    rep = h // hkv
    kk, vv = k.double().repeat_interleave(rep, 1), v.double().repeat_interleave(rep, 1)
    s = torch.einsum("nhd,shd->hns", q.double(), kk) / math.sqrt(d)
    qpos = torch.arange(total - n, total)[:, None]
    kpos = torch.arange(total)[None, :]
    s = s.masked_fill(~((kpos <= qpos) & (kpos > qpos - window)), float("-inf"))
    return torch.einsum("hns,shd->nhd", torch.softmax(s, -1), vv).reshape(n, h * d)


def _batch(past, now, enc, nh, nkv, d, bs, seed):
    """A mixed batch over a shuffled block pool; returns the block_attention arguments and every sequence's full K / V."""
    g = torch.Generator().manual_seed(seed)
    nseq = len(now)
    totals = [p + n for p, n in zip(past, now)]
    nblk = [(t + bs - 1) // bs for t in totals]
    perm = torch.randperm(sum(nblk) + 3, generator=g).tolist()
    mb = max(nblk)
    bt = torch.zeros(nseq, mb, dtype=torch.int32)
    kc = torch.full((len(perm), nkv, bs, d), float("nan"))
    vc = torch.full_like(kc, float("nan"))
    K, V, o = [], [], 0
    for b in range(nseq):
        bt[b, :nblk[b]] = torch.tensor(perm[o:o + nblk[b]], dtype=torch.int32)
        o += nblk[b]
        K.append(torch.randn(totals[b], nkv, d, generator=g))
        V.append(torch.randn(totals[b], nkv, d, generator=g))
        for p in range(past[b]):                                  # the cached prefix
            kc[bt[b, p // bs], :, p % bs] = K[b][p]
            vc[bt[b, p // bs], :, p % bs] = V[b][p]
    cu = torch.tensor([0] + list(torch.cumsum(torch.tensor(now), 0).tolist()), dtype=torch.int32)
    qkv = torch.zeros(int(cu[-1]), (nh + 2 * nkv) * d)
    Q = []
    for b in range(nseq):
        q = torch.randn(now[b], nh, d, generator=g)
        Q.append(q)
        qkv[cu[b]:cu[b + 1]] = torch.cat([q, K[b][past[b]:], V[b][past[b]:]], 1).reshape(now[b], (nh + 2 * nkv) * d)
    dec = torch.tensor([0 if e else p for p, e in zip(past, enc)], dtype=torch.int32)
    args = (qkv, kc, vc, torch.tensor(enc, dtype=torch.int32), dec, torch.tensor(now, dtype=torch.int32), cu, bt, bs)
    return args, Q, K, V, cu


@pytest.mark.parametrize("window", [1, 3, 8, 13, 10_000])   # 1, below the block size, a multiple of it, not a multiple, past every context
def test_reference_window_matches_dense_masked_attention(window):
    nh, nkv, d, bs = 4, 2, 16, 8
    past = [0, 30, 21, 17, 40, 9]
    now = [12, 1, 3, 0, 9, 1]                                     # prefill, decode, verify, empty, continuing chunk, decode
    enc = [12, 0, 0, 0, 0, 0]
    args, Q, K, V, cu = _batch(past, now, enc, nh, nkv, d, bs, seed=window)
    qkv, kc, vc, bt = args[0], args[1], args[2], args[7]
    # blocks wholly below each sequence's window are never read: poison them
    for b in range(len(now)):
        lo = max(0, past[b] - window + 1)
        for j in range(lo // bs):
            kc[bt[b, j]] = float("nan")
            vc[bt[b, j]] = float("nan")
    out = _block_attention_ref(*args, sliding_window=window)[0].as_subclass(torch.Tensor)
    for b in range(len(now)):
        if now[b] == 0:
            continue
        ref = _dense(Q[b], K[b], V[b], window)
        torch.testing.assert_close(out[cu[b]:cu[b + 1]].double(), ref, rtol=1e-5, atol=1e-5)
        assert not torch.isnan(out[cu[b]:cu[b + 1]]).any()


def test_window_past_the_context_equals_no_window():
    args, *_ = _batch([0, 20, 11], [7, 1, 4], [7, 0, 0], 4, 4, 16, 4, seed=3)
    args2 = tuple(a.clone() if isinstance(a, torch.Tensor) else a for a in args)
    a = _block_attention_ref(*args, sliding_window=1000)[0]
    b = _block_attention_ref(*args2)[0]
    assert torch.equal(a.as_subclass(torch.Tensor), b.as_subclass(torch.Tensor))


@pytest.mark.parametrize("bad", [0, -3, 2.5, True])
def test_sliding_window_argument_errors(bad):
    args, *_ = _batch([0], [4], [4], 2, 2, 16, 4, seed=0)
    with pytest.raises(ValueError, match="sliding_window"):
        block_attention(*args, sliding_window=bad)
    with pytest.raises(ValueError, match="sliding_window"):
        _block_attention_ref(*args, sliding_window=bad)


def test_sliding_window_with_shared_prefix_is_rejected():
    args, *_ = _batch([0], [4], [4], 2, 2, 16, 4, seed=0)
    with pytest.raises(ValueError, match="shared_prefix"):
        block_attention(*args, shared_prefix=([0, 1], [0], [4]), sliding_window=4)


def test_mistral_config():
    cfg = models.mistral_7b()
    assert (cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers) == (4096, 14336, 32)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.sliding_window, cfg.head_dim) == (32, 8, 4096, 128)
    assert models.MixtralConfig(sliding_window=7).sliding_window == 7
    assert models.llama_tiny().sliding_window is None


def _model(seed=0, **kw):
    paddle.seed(seed)
    cfg = models.llama_tiny(**kw)
    m = models.LlamaForCausalLM(cfg)
    m.eval()
    return m, cfg


def test_llama_window_forward_matches_explicit_mask():
    window, n = 5, 19
    m, cfg = _model(0, sliding_window=window, num_key_value_heads=2)
    at = m.llama.layers[0].self_attn
    nh, nkv, hd = at.num_heads, at.num_kv_heads, at.head_dim
    h = torch.randn(2, n, cfg.hidden_size, generator=torch.Generator().manual_seed(0))
    cos, sin = models.llama.rope_cache(cfg, h.device)
    qkv = at.qkv_proj(h)
    with torch.no_grad():
        got = at.attend(qkv.clone(), cos, sin).as_subclass(torch.Tensor)
        # explicit-mask reference on the same rotated projection
        x = models.llama.KR.apply_rope_packed(qkv.clone(), cos, sin, nh + nkv, nh + 2 * nkv, hd, None, neox=True).as_subclass(torch.Tensor)
        x = x.reshape(2, n, nh + 2 * nkv, hd)
        q, k, v = x[:, :, :nh], x[:, :, nh:nh + nkv].repeat_interleave(nh // nkv, 2), x[:, :, nh + nkv:].repeat_interleave(nh // nkv, 2)
        mask = models.llama.window_mask(n, n, window, h.device)
        o = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=mask)
        ref = at.o_proj(o.transpose(1, 2).reshape(2, n, nh * hd)).as_subclass(torch.Tensor)
    torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-5)
    # the window changes the logits once the context passes it
    ids = torch.randint(1, cfg.vocab_size, (2, n), generator=torch.Generator().manual_seed(1))
    full, _ = _model(0, num_key_value_heads=2)
    with torch.no_grad():
        assert not torch.allclose(m(ids).as_subclass(torch.Tensor), full(ids).as_subclass(torch.Tensor))


def _alone(m, prompt, n):
    out = models.generate(m, torch.tensor([prompt]), max_new_tokens=n).as_subclass(torch.Tensor)
    return out[0, len(prompt):].tolist()


def _prompts(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]


class _Watch:
    """Runs an engine step by step and checks, after every step, the blocks each fully prefilled sequence holds."""

    def __init__(self, eng, window):
        self.eng, self.cap = eng, -(-window // eng.block_size) + 2

    def run(self):
        while self.eng.has_unfinished():
            self.eng.step()
            for s in self.eng.running:
                if s.cached >= s.target:
                    assert len(s.owned()) <= self.cap, (s.id, s.cached, s.blocks)
                    assert all(b == -1 for b in s.blocks[:s.released])
        return {i: s.generated for i, s in self.eng.done.items()}


@pytest.mark.parametrize("chunk", [None, 5])
def test_engine_window_matches_generate_and_releases_blocks(chunk):
    window, bs = 7, 4
    m, cfg = _model(1, sliding_window=window, num_key_value_heads=2)
    prompts = _prompts(cfg, (5, 17, 9, 23), seed=1)
    news = [14, 9, 16, 6]
    eng = models.LLMEngine(m, num_blocks=64, block_size=bs, max_batch_tokens=32, max_prefill_chunk=chunk)
    ids = [eng.add_request(p, n) for p, n in zip(prompts, news)]
    res = _Watch(eng, window).run()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n), i
    assert eng.stats["released_blocks"] > 0
    assert eng.alloc.num_free() == 64


def test_engine_window_under_preemption():
    window, bs = 12, 4
    m, cfg = _model(2, sliding_window=window)
    prompts = _prompts(cfg, (6, 11, 9), seed=2)
    eng = models.LLMEngine(m, num_blocks=9, block_size=bs, max_batch_tokens=10, max_prefill_chunk=3)
    ids = [eng.add_request(p, 14) for p in prompts]
    res = _Watch(eng, window).run()
    assert eng.stats["preemptions"] >= 1 and eng.stats["released_blocks"] > 0
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 14)
    assert eng.alloc.num_free() == 9


def test_engine_window_with_a_draft():
    m, cfg = _model(3, sliding_window=6)
    draft, _ = _model(4, sliding_window=6, num_hidden_layers=1)
    prompts = _prompts(cfg, (7, 12), seed=3)
    eng = models.LLMEngine(m, num_blocks=48, block_size=4, draft_model=draft, num_speculative_tokens=3)
    ids = [eng.add_request(p, 12) for p in prompts]
    res = _Watch(eng, 6).run()
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 12)
    assert eng.stats["released_blocks"] > 0
    # a draft without a window keeps every block
    plain, _ = _model(4, num_hidden_layers=1)
    eng = models.LLMEngine(m, num_blocks=48, block_size=4, draft_model=plain, num_speculative_tokens=2)
    i = eng.add_request(prompts[1], 10)
    assert eng.run_until_done()[i] == _alone(m, prompts[1], 10)
    assert eng.stats["released_blocks"] == 0


def test_engine_window_rejects_prefix_caching():
    m, _ = _model(sliding_window=4)
    with pytest.raises(ValueError, match="prefix_caching"):
        models.LLMEngine(m, num_blocks=8, block_size=4, enable_prefix_caching=True)


@pytest.mark.skipif(shutil.which("cuobjdump") is None or not all(os.path.exists(o) for o in WINDOW_OBJS),
                    reason="cuobjdump or the built objects are missing")
def test_windowed_launches_use_no_local_memory_and_keep_wgmma_pipelined():
    funcs = {}
    for obj in WINDOW_OBJS:
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
        for f in re.split(r"\n\s*Function : ", sass)[1:]:
            name, body = f.split("\n", 1)
            funcs[name.strip()] = body
    # the kernels a windowed call launches, by mangled name: windowed verify splits carry WINDOW = true (Lb1E) after the head size, and
    # windowed decode and verify merge their splits with the unwindowed merge kernels
    kinds = {"decode_split_window_kernel": lambda n: "decode_split_window_kernel" in n,
             "decode_split_q8_window_kernel": lambda n: "decode_split_q8_window_kernel" in n,
             "decode_merge_kernel": lambda n: "decode_merge_kernel" in n,
             "multi_split_kernel (WINDOW)": lambda n: "multi_split_kernel" in n and re.search(r"Li(64|128)ELb1E", n) is not None,
             "multi_merge_kernel": lambda n: "multi_merge_kernel" in n,
             "paged_work_window_kernel": lambda n: "paged_work_window_kernel" in n,
             "fwd_window_kernel": lambda n: "fwd_window_kernel" in n}
    counts = {"decode_split_window_kernel": 4, "decode_split_q8_window_kernel": 4, "decode_merge_kernel": 4, "multi_split_kernel (WINDOW)": 8,
              "multi_merge_kernel": 4, "paged_work_window_kernel": 1, "fwd_window_kernel": 8}
    for k, n in counts.items():
        assert sum(kinds[k](name) for name in funcs) == n, (k, sorted(funcs))
    for name, body in funcs.items():
        if not any(is_kind(name) for is_kind in kinds.values()):
            continue
        assert not re.search(r"\b(LDL|STL)\b", body), name
        if "fwd_window_kernel" in name:
            mma = len(re.findall(r"\bHGMMA\.", body))
            assert 0 < body.count("WARPGROUP.ARRIVE") < mma, name
