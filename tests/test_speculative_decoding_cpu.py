"""models.LLMEngine(draft_model=..., num_speculative_tokens=k): a draft model proposes up to k tokens per greedy decode sequence and one
target forward verifies them; greedy tokens equal isolated generation whatever the draft, under mid-flight arrivals, chunked prefill,
preemption, eos and sampling requests, and every block goes back to the pool."""
import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models


def _model(seed=0, **kw):
    paddle.seed(seed)
    cfg = models.llama_tiny(**kw)
    m = models.LlamaForCausalLM(cfg)
    m.eval()
    return m, cfg


def _alone(m, prompt, n):
    out = models.generate(m, torch.tensor([prompt]), max_new_tokens=n).as_subclass(torch.Tensor)
    return out[0, len(prompt):].tolist()


def _prompts(cfg, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in lens]


@pytest.mark.parametrize("k", [1, 3, 5])
def test_draft_equal_to_target_accepts_every_proposal(k):
    m, cfg = _model()
    prompt = _prompts(cfg, (9,), seed=0)[0]
    n = 13
    eng = models.LLMEngine(m, num_blocks=16, block_size=4, draft_model=m, num_speculative_tokens=k)
    rid = eng.add_request(prompt, n)
    res = eng.run_until_done()
    assert res[rid] == _alone(m, prompt, n)
    assert eng.stats["draft_tokens"] > 0 and eng.stats["accepted_tokens"] == eng.stats["draft_tokens"]
    assert eng.stats["steps"] == 1 + -(-(n - 1) // (k + 1))          # the prefill step, then k + 1 tokens per step
    assert eng.stats["decode_tokens"] == n - 1
    assert eng.alloc.num_free() == 16


@pytest.mark.parametrize("draft_kw", [dict(seed=7), dict(seed=3, num_hidden_layers=1, num_key_value_heads=2)])
def test_other_drafts_keep_the_target_tokens(draft_kw):
    m, cfg = _model()
    seed = draft_kw.pop("seed")
    d, _ = _model(seed, **draft_kw)
    prompts = _prompts(cfg, (5, 17, 9, 3), seed=1)
    news = [9, 6, 11, 7]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, draft_model=d, num_speculative_tokens=3)
    ids = [eng.add_request(p, n) for p, n in zip(prompts, news)]
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n)
    assert 0 <= eng.stats["accepted_tokens"] < eng.stats["draft_tokens"]
    assert eng.alloc.num_free() == 64


@pytest.mark.parametrize("chunk", [None, 3])
def test_mid_flight_arrivals_and_chunked_prefill(chunk):
    m, cfg = _model()
    d, _ = _model(5, num_hidden_layers=1)
    prompts = _prompts(cfg, (5, 17, 9, 3, 22), seed=2)
    news = [6, 4, 8, 5, 7]                                           # none a multiple of k + 1 = 4
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, max_batch_tokens=12 if chunk else 64, max_prefill_chunk=chunk, draft_model=d,
                           num_speculative_tokens=3)
    ids = [eng.add_request(prompts[0], news[0]), eng.add_request(prompts[1], news[1])]
    eng.step()
    eng.step()
    ids.append(eng.add_request(prompts[2], news[2]))                 # arrives while others decode (and, chunked, prefill)
    eng.step()
    ids += [eng.add_request(prompts[3], news[3]), eng.add_request(prompts[4], news[4])]
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n), (i, res[i])
    assert eng.stats["prefill_tokens"] == sum(len(p) for p in prompts)
    assert eng.alloc.num_free() == 64


def test_preemption_with_speculation():
    m, cfg = _model(seed=1)
    prompts = _prompts(cfg, (6, 11, 9), seed=1)
    eng = models.LLMEngine(m, num_blocks=9, block_size=4, draft_model=m, num_speculative_tokens=2)
    ids = [eng.add_request(p, 10) for p in prompts]
    res = eng.run_until_done()
    assert eng.stats["preemptions"] >= 1
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 10)
    assert eng.alloc.num_free() == 9


def test_eos_inside_an_accepted_run():
    m, cfg = _model()
    prompt = _prompts(cfg, (7,), seed=3)[0]
    ref = _alone(m, prompt, 12)
    eos = ref[3]                                                      # the 4th token: inside the first verify step's run of 6
    cut = ref[:ref.index(eos) + 1]
    eng = models.LLMEngine(m, num_blocks=16, block_size=4, draft_model=m, num_speculative_tokens=5)
    rid = eng.add_request(prompt, 12, eos_token_id=eos)
    first = eng.step()
    second = eng.step()
    assert [t for _, t, _ in first + second] == cut and second[-1][2]
    assert eng.result(rid).as_subclass(torch.Tensor).tolist() == cut
    assert eng.alloc.num_free() == 16


def test_sampling_requests_do_not_speculate():
    m, cfg = _model()
    prompts = _prompts(cfg, (5, 8, 6), seed=4)
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, draft_model=m, num_speculative_tokens=3)
    greedy = [eng.add_request(prompts[0], 9), eng.add_request(prompts[2], 5)]
    paddle.seed(11)
    sampled = eng.add_request(prompts[1], 9, do_sample=True, temperature=0.8, top_k=20)
    counts = {}
    while eng.has_unfinished():
        for i, _, _ in eng.step():
            counts.setdefault(i, []).append(eng.stats["steps"])
    res = {i: s.generated for i, s in eng.done.items()}
    assert res[greedy[0]] == _alone(m, prompts[0], 9) and res[greedy[1]] == _alone(m, prompts[2], 5)
    assert len(res[sampled]) == 9 and counts[sampled] == list(range(1, 10))   # one token every step
    assert eng.stats["accepted_tokens"] == eng.stats["draft_tokens"] > 0
    assert eng.alloc.num_free() == 64


def test_short_pool_shrinks_speculation_without_preempting():
    m, cfg = _model()
    prompts = _prompts(cfg, (8, 8), seed=5)
    eng = models.LLMEngine(m, num_blocks=7, block_size=4, draft_model=m, num_speculative_tokens=5)
    a, b = [eng.add_request(p, 12) for p in prompts]
    eng.step()                                                        # both prompts: 3 blocks each, 1 free
    eng.step()                                                        # a takes the free block for 5 proposals, b is left 3
    seqs = {s.id: s for s in eng.running}
    assert eng.stats["preemptions"] == 0
    assert eng.stats["draft_tokens"] == 5 + 3
    assert len(seqs[a].generated) == 1 + 6 and len(seqs[b].generated) == 1 + 4
    res = eng.run_until_done()
    assert res[a] == _alone(m, prompts[0], 12) and res[b] == _alone(m, prompts[1], 12)
    assert eng.alloc.num_free() == 7


def test_invalid_speculation_arguments():
    m, cfg = _model()
    d, _ = _model(1, vocab_size=256)
    with pytest.raises(ValueError):
        models.LLMEngine(m, draft_model=m)                            # no k
    with pytest.raises(ValueError):
        models.LLMEngine(m, num_speculative_tokens=3)                 # no draft
    with pytest.raises(ValueError):
        models.LLMEngine(m, draft_model=m, num_speculative_tokens=-1)
    with pytest.raises(ValueError):
        models.LLMEngine(m, draft_model=d, num_speculative_tokens=2)  # vocab 256 vs 512


def test_no_draft_keeps_the_stats():
    m, cfg = _model()
    prompts = _prompts(cfg, (5, 11), seed=6)
    runs = []
    for kw in ({}, dict(draft_model=None, num_speculative_tokens=0)):
        eng = models.LLMEngine(m, num_blocks=32, block_size=4, **kw)
        ids = [eng.add_request(p, 6) for p in prompts]
        res = eng.run_until_done()
        runs.append(([res[i] for i in ids], dict(eng.stats)))
    assert runs[0] == runs[1]
    assert set(runs[0][1]) == {"steps", "prefill_tokens", "decode_tokens", "preemptions", "max_running"}
