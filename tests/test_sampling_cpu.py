"""Token sampling on CPU (kernels.sampling.sample_ref, the CUDA kernel's oracle): the Philox stream, the by-value rules, the draw's
distribution, paddle.top_p_sampling, LLMEngine's seeded, batched sampling, and the kernel's sm_90a register report (no spills)."""
import os
import re
import shutil
import subprocess

import pytest
import torch
from scipy import stats

import paddle_b200 as paddle
from paddle_b200 import models
from paddle_b200.kernels import sampling


def _params(rows, temperature=1.0, top_k=0, top_p=1.0, seed=0, offset=0):
    col = lambda v, dt: (v.to(dt) if isinstance(v, torch.Tensor) else torch.full((rows,), v, dtype=dt))
    return (col(temperature, torch.float32), col(top_k, torch.int32), col(top_p, torch.float32), col(seed, torch.int64),
            col(offset, torch.int64))


def _draws(x, n, **kw):
    """ids of one row x [vocab] under seeds 0 .. n-1"""
    xs = x.reshape(1, -1).expand(n, -1).contiguous()
    thr = kw.pop("threshold", None)
    trunc = kw.pop("truncated", True)
    is_prob = kw.pop("is_prob", False)
    return sampling.sample(xs, *_params(n, seed=torch.arange(n), **kw), threshold=None if thr is None else torch.full((n,), thr),
                           is_prob=is_prob, truncated=trunc)[0]


def test_philox_known_answers():
    m = 0xFFFFFFFF
    assert [int(w) for w in sampling.philox4x32_10(0, 0, 0, 0, 0, 0)] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    assert [int(w) for w in sampling.philox4x32_10(m, m, m, m, m, m)] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
    u = sampling.uniforms(7, 3, 64)
    assert ((u > 0) & (u < 1)).all() and len(set(u.tolist())) == 64


def test_top1_and_tiny_top_p_give_the_argmax():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(64, 1000, generator=g)
    want = x.argmax(-1)
    for kw in (dict(top_k=1), dict(top_p=1e-6), dict(temperature=0.0), dict(temperature=0.5, top_k=1, top_p=0.3)):
        assert torch.equal(sampling.sample(x, *_params(64, seed=torch.arange(64), **kw))[0], want), kw


def test_greedy_ties_take_the_lowest_index():
    x = torch.tensor([[1.0, 3.0, 0.0, 3.0, 3.0], [-0.0, 0.0, -1.0, 0.0, -2.0]])
    assert sampling.sample(x, *_params(2, temperature=0.0))[0].tolist() == [1, 0]


def test_top_k_keeps_ties():
    x = torch.tensor([5.0, 5.0, 5.0, 1.0, 0.0, 4.9])
    got = set(_draws(x, 400, top_k=1).tolist())
    assert got == {0, 1, 2}
    assert set(_draws(x, 400, top_k=3).tolist()) == {0, 1, 2}


def test_top_p_boundary_follows_the_value_rule():
    p = torch.tensor([0.4, 0.3, 0.3, 0.0])                 # tokens 1 and 2 tie across the boundary
    assert set(_draws(p, 600, top_p=0.5, is_prob=True).tolist()) == {0, 1, 2}
    assert set(_draws(p, 600, top_p=0.35, is_prob=True).tolist()) == {0}
    logits = p.clamp(min=1e-9).log()
    assert set(_draws(logits, 600, top_p=0.5).tolist()) == {0, 1, 2}
    assert set(_draws(logits, 600, top_p=0.39).tolist()) == {0}


def test_threshold_modes():
    p = torch.tensor([0.5, 0.3, 0.2])
    n = 4000
    nt = _draws(p, n, is_prob=True, threshold=0.25, truncated=False)
    tr = _draws(p, n, is_prob=True, threshold=0.25, truncated=True)
    assert set(nt.tolist()) == {0, 1} and set(tr.tolist()) == {0, 1}
    assert abs((nt == 1).float().mean().item() - 0.3 / 0.8) < 0.03       # token 2 left the race
    assert abs((tr == 1).float().mean().item() - 0.5) < 0.03             # draws of token 2 fall back to token 1
    for trunc in (True, False):                                           # the top-1 is returned even below the threshold
        assert set(_draws(p, 200, is_prob=True, threshold=0.9, truncated=trunc).tolist()) == {0}


def test_return_top_equals_topk():
    g = torch.Generator().manual_seed(1)
    x = torch.rand(5, 300, generator=g)
    _, _, tv, ti = sampling.sample(x, *_params(5), is_prob=True, k_out=7)
    ref = torch.topk(x, 7)
    assert torch.equal(tv, ref.values) and torch.equal(ti, ref.indices)
    with pytest.raises(ValueError):
        sampling.sample(x, *_params(5), k_out=301)


def test_a_row_does_not_depend_on_its_batch():
    g = torch.Generator().manual_seed(2)
    x = torch.randn(12, 500, generator=g)
    prm = _params(12, temperature=torch.rand(12, generator=g) + 0.3, top_k=torch.tensor([0, 5, 50] * 4), top_p=torch.tensor([1.0, 0.9, 0.5] * 4),
                  seed=torch.arange(12) * 7919, offset=torch.arange(12) + 100)
    ids = sampling.sample(x, *prm)[0]
    perm = torch.randperm(12, generator=g)
    assert torch.equal(sampling.sample(x[perm], *(p[perm] for p in prm))[0], ids[perm])
    assert torch.equal(sampling.sample(x[3:5], *(p[3:5] for p in prm))[0], ids[3:5])


def test_draw_distribution_chi_square():
    logits = torch.tensor([2.0, 1.5, 1.0, 0.7, 0.3, 0.0, -0.5, -1.0])
    T, k, p, n = 0.8, 6, 0.9, 20000
    probs = torch.softmax(logits.double() / T, -1)
    probs[k:] = 0                                          # values are distinct and descending: top_k keeps the first k
    probs /= probs.sum()
    keep = (probs.cumsum(0) - probs) <= p
    probs = torch.where(keep, probs, torch.zeros_like(probs))
    probs /= probs.sum()
    ids = _draws(logits, n, temperature=T, top_k=k, top_p=p)
    counts = torch.bincount(ids, minlength=8).double()
    live = probs > 0
    assert counts[~live].sum() == 0
    chi = stats.chisquare(counts[live].numpy(), (probs[live] * n).numpy())
    assert chi.pvalue > 1e-3, chi


def test_top_p_sampling_api():
    p = torch.tensor([[0.5, 0.3, 0.2, 0.0], [0.1, 0.1, 0.1, 0.7]])
    out, ids = paddle.top_p_sampling(paddle.to_tensor(p), paddle.to_tensor(torch.tensor([0.6, 0.5])), seed=3)
    assert list(ids.shape) == [2, 1] and list(out.shape) == [2, 1] and ids.dtype == torch.int64
    assert int(ids[1, 0]) == 3 and float(out[1, 0]) == pytest.approx(0.7)
    a = paddle.top_p_sampling(paddle.to_tensor(p), paddle.to_tensor(torch.tensor([0.9, 0.9])), topp_seed=paddle.to_tensor(torch.tensor([5, 6])))[1]
    b = paddle.top_p_sampling(paddle.to_tensor(p), paddle.to_tensor(torch.tensor([0.9, 0.9])), topp_seed=paddle.to_tensor(torch.tensor([5, 6])))[1]
    assert torch.equal(a, b)
    _, _, tv, ti = paddle.top_p_sampling(paddle.to_tensor(p), paddle.to_tensor(torch.tensor([0.9, 0.9])), k=2, return_top=True)
    ref = torch.topk(p, 2)
    assert torch.equal(torch.as_tensor(tv), ref.values) and torch.as_tensor(ti).tolist() == [[0, 1], [3, 0]]   # ties: lowest index
    with pytest.raises(ValueError):
        paddle.top_p_sampling(paddle.to_tensor(p), paddle.to_tensor(torch.tensor([0.9, 0.9])), mode="bogus")
    with pytest.raises(ValueError):
        paddle.top_p_sampling(paddle.to_tensor(p), paddle.to_tensor(torch.tensor([0.9, 0.9])), return_top=True)


# ---- LLMEngine ----------------------------------------------------------------------------------------------------------------------
def _model(seed=0, **kw):
    paddle.seed(seed)
    cfg = models.llama_tiny(**kw)
    m = models.LlamaForCausalLM(cfg)
    m.eval()
    return m, cfg


SAMPLED = dict(do_sample=True, temperature=0.8, top_k=20, top_p=0.95)


def _prompts(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]


def _seeded_alone(m, prompt, n, seed, **kw):
    eng = models.LLMEngine(m, num_blocks=64, block_size=4)
    i = eng.add_request(prompt, n, seed=seed, **SAMPLED)
    return eng.run_until_done()[i]


def test_seeded_request_alone_and_in_a_batch():
    m, cfg = _model()
    ps = _prompts(cfg, (6, 11, 4, 9), 0)
    alone = _seeded_alone(m, ps[0], 8, seed=1234)
    assert alone != _seeded_alone(m, ps[0], 8, seed=99)
    eng = models.LLMEngine(m, num_blocks=64, block_size=4)
    others = [eng.add_request(p, 6, **SAMPLED) for p in ps[1:3]]
    eng.step()
    i = eng.add_request(ps[0], 8, seed=1234, **SAMPLED)      # joins mid-flight, next to unseeded sampled and greedy requests
    eng.add_request(ps[3], 5)
    res = eng.run_until_done()
    assert res[i] == alone and all(len(res[o]) == 6 for o in others)


def test_seeded_request_under_preemption_chunking_and_prefix_hits():
    m, cfg = _model(1)
    ps = _prompts(cfg, (6, 6, 6), 1)
    alone = [_seeded_alone(m, p, 10, seed=10 + j) for j, p in enumerate(ps)]
    eng = models.LLMEngine(m, num_blocks=7, block_size=4)
    ids = [eng.add_request(p, 10, seed=10 + j, **SAMPLED) for j, p in enumerate(ps)]
    res = eng.run_until_done()
    assert eng.stats["preemptions"] >= 1 and [res[i] for i in ids] == alone
    long = _prompts(cfg, (19,), 2)[0]
    want = _seeded_alone(m, long, 6, seed=5)
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, max_batch_tokens=12, max_prefill_chunk=5)
    i = eng.add_request(long, 6, seed=5, **SAMPLED)
    assert eng.run_until_done()[i] == want
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, enable_prefix_caching=True)
    a = eng.add_request(long, 6, seed=5, **SAMPLED)
    eng.run_until_done()
    b = eng.add_request(long, 6, seed=5, **SAMPLED)
    res = eng.run_until_done()
    assert eng.stats["prefix_hit_tokens"] > 0 and res[a] == want and res[b] == want


def test_seeded_request_with_a_draft_model_and_one_call_per_step(monkeypatch):
    m, cfg = _model(2)
    ps = _prompts(cfg, (5, 8, 7), 3)
    want = _seeded_alone(m, ps[0], 7, seed=77)
    calls = []
    real = sampling.sample

    def counting(x, *a, **k):
        calls.append(x.shape[0])
        return real(x, *a, **k)

    monkeypatch.setattr(sampling, "sample", counting)
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, draft_model=m, num_speculative_tokens=3)
    i = eng.add_request(ps[0], 7, seed=77, **SAMPLED)
    greedy = [eng.add_request(p, 6) for p in ps[1:]]
    steps, per_step = 0, []
    while eng.has_unfinished():
        n = len(calls)
        out = eng.step()
        steps += 1
        per_step.append(len(calls) - n)
        assert sum(1 for rid, _, _ in out if rid == i) <= 1           # a sampled request decodes one token per step
    res = {j: eng.done[j].generated for j in eng.done}
    assert res[i] == want and per_step == [1] * steps and max(calls) > 3
    assert eng.stats["accepted_tokens"] > 0
    for j, p in zip(greedy, ps[1:]):
        assert res[j] == models.generate(m, torch.tensor([p]), max_new_tokens=6).as_subclass(torch.Tensor)[0, len(p):].tolist()


def test_unseeded_requests_follow_paddle_seed():
    m, cfg = _model(3)
    p = _prompts(cfg, (5,), 4)[0]
    runs = []
    for _ in range(2):
        paddle.seed(11)
        eng = models.LLMEngine(m, num_blocks=32, block_size=4)
        i = eng.add_request(p, 6, **SAMPLED)
        runs.append(eng.run_until_done()[i])
    assert runs[0] == runs[1]


def _nvcc():
    from torch.utils.cpp_extension import CUDA_HOME

    path = os.path.join(CUDA_HOME, "bin", "nvcc") if CUDA_HOME else shutil.which("nvcc")
    return path if path and os.path.exists(path) else None


@pytest.mark.skipif(_nvcc() is None, reason="nvcc not found")
def test_kernel_compiles_without_spills():
    csrc = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "paddle_b200", "csrc")
    r = subprocess.run([_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-Xptxas", "-v",
                        "-I", csrc, "-c", os.path.join(csrc, "sampling.cu"), "-o", os.devnull], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    frames = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stderr)
    assert len(frames) >= 7 and all(f == ("0", "0", "0") for f in frames), r.stderr
