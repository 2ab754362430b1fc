"""models.LLMEngine(max_prefill_chunk=N): prompts are prefilled over several steps, each chunk attending to the chunks already in the
paged cache; greedy tokens equal isolated generation, a prompt longer than max_batch_tokens is served, and None keeps the old schedule."""
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


@pytest.mark.parametrize("chunk", [3, 7])
def test_chunked_prefill_matches_isolated_generation(chunk):
    m, cfg = _model()
    prompts = _prompts(cfg, (5, 17, 9, 3, 22), seed=0)     # lengths straddle the chunk and the 4-token block edges
    news = [6, 4, 8, 5, 3]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, max_batch_tokens=12, max_prefill_chunk=chunk)
    ids = [eng.add_request(prompts[0], news[0]), eng.add_request(prompts[1], news[1])]
    first = eng.step()
    assert all(i != ids[1] for i, _, _ in first)               # the 17-token prompt is still being prefilled
    eng.step()
    ids.append(eng.add_request(prompts[2], news[2]))            # arrives while others decode and prefill
    eng.step()
    ids.append(eng.add_request(prompts[3], news[3]))
    ids.append(eng.add_request(prompts[4], news[4]))
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n), (i, res[i])
    assert eng.alloc.num_free() == 64
    assert eng.stats["prefill_tokens"] == sum(len(p) for p in prompts)


@pytest.mark.parametrize("chunk", [3, 7])
def test_chunked_prefill_with_preemption(chunk):
    m, cfg = _model(seed=1)
    prompts = _prompts(cfg, (6, 11, 9), seed=1)
    eng = models.LLMEngine(m, num_blocks=9, block_size=4, max_batch_tokens=10, max_prefill_chunk=chunk)
    ids = [eng.add_request(p, 10) for p in prompts]
    res = eng.run_until_done()
    assert eng.stats["preemptions"] >= 1
    for i, p in zip(ids, prompts):
        assert res[i] == _alone(m, p, 10)
    assert eng.alloc.num_free() == 9


def test_preempting_a_half_prefilled_sequence_restarts_it():
    m, cfg = _model(seed=3)
    p0, p1 = _prompts(cfg, (4, 14), seed=3)
    eng = models.LLMEngine(m, num_blocks=6, block_size=4, max_batch_tokens=6, max_prefill_chunk=3)
    a = eng.add_request(p0, 9)                                  # 4 + 9 tokens: 4 blocks when it has grown
    eng.step()
    b = eng.add_request(p1, 2)                                  # 14 + 2 tokens: 4 blocks; admitted only when a frees its own
    seen_partial = False
    while eng.has_unfinished():
        eng.step()
        s = next((x for x in eng.running if x.id == b), None)
        seen_partial |= s is not None and 0 < s.cached < s.target
    res = {i: s.generated for i, s in eng.done.items()}
    assert seen_partial
    assert res[a] == _alone(m, p0, 9) and res[b] == _alone(m, p1, 2)
    assert eng.alloc.num_free() == 6


def test_prompt_longer_than_the_token_budget_completes():
    m, cfg = _model(seed=2)
    (p,) = _prompts(cfg, (23,), seed=2)
    eng = models.LLMEngine(m, num_blocks=16, block_size=4, max_batch_tokens=8)
    eng.add_request(p, 4)
    with pytest.raises(MemoryError):                            # without chunking it can never be scheduled
        eng.step()
    eng = models.LLMEngine(m, num_blocks=16, block_size=4, max_batch_tokens=8, max_prefill_chunk=64)
    i = eng.add_request(p, 4)
    res = eng.run_until_done()
    assert res[i] == _alone(m, p, 4)
    assert eng.stats["steps"] == 3 + 3                          # 23 tokens in chunks of at most 8, then three decode steps


def test_no_chunk_keeps_the_schedule():
    m, cfg = _model(seed=4)
    prompts = _prompts(cfg, (5, 17, 9, 3), seed=4)
    runs = []
    for kw in ({}, {"max_prefill_chunk": None}, {"max_prefill_chunk": 1000}):
        eng = models.LLMEngine(m, num_blocks=12, block_size=4, max_batch_tokens=24, **kw)
        ids = [eng.add_request(p, 6) for p in prompts]
        res = eng.run_until_done()
        runs.append((dict(eng.stats), [res[i] for i in ids]))
    assert runs[0] == runs[1]
    assert runs[2][1] == runs[0][1]                             # chunks larger than every prompt change nothing either
    with pytest.raises(ValueError):
        models.LLMEngine(m, num_blocks=4, block_size=4, max_prefill_chunk=0)
