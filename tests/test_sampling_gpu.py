"""The sm_90a sampling kernel (csrc/sampling.cu) against kernels.sampling.sample_ref, its Philox draws, paddle.top_p_sampling on CUDA
against its CPU path, and LLMEngine's batched sampling on the GPU (needs a GPU)."""
import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models
from paddle_b200._build import ext
from paddle_b200.kernels import sampling

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
VOCABS = [1000, 32000, 128256, 152064]


def _mixed_params(rows, g):
    """Row r cycles through greedy, temperature only, top_k, top_p, top_k + top_p; seeds and offsets differ per row."""
    mode = torch.arange(rows) % 5
    temp = torch.where(mode == 0, torch.zeros(rows), 0.5 + torch.rand(rows, generator=g))
    top_k = torch.where((mode == 2) | (mode == 4), torch.randint(1, 200, (rows,), generator=g), torch.zeros(rows, dtype=torch.long))
    top_p = torch.where((mode == 3) | (mode == 4), 0.2 + 0.75 * torch.rand(rows, generator=g), torch.ones(rows))
    seed = torch.randint(-2 ** 62, 2 ** 62, (rows,), generator=g)
    offset = torch.randint(0, 2 ** 40, (rows,), generator=g)
    return mode, [temp.float(), top_k.int(), top_p.float(), seed, offset]


def _compare(x, prm, mode, threshold=None, is_prob=False, truncated=True):
    """Kernel ids against the reference's; a mismatch is excused only in a row whose top-p boundary mass lies within 1e-5 of top_p or
    whose top two race keys lie within 1e-6 (relative), and never in a greedy or top_k-only row.  Returns the excused rows."""
    dev = [p.cuda() for p in prm]
    got = sampling.sample(x, *dev, threshold=None if threshold is None else threshold.cuda(), is_prob=is_prob, truncated=truncated)
    ids, vals = got[0].cpu(), got[1]
    assert torch.equal(vals.cpu(), x.cpu().gather(1, ids.reshape(-1, 1)).reshape(-1))
    ref, race, mass, greedy, p_on = sampling.race_parts(x.cpu(), *prm, threshold=threshold, is_prob=is_prob, truncated=truncated)
    bad = (ids != ref).nonzero().reshape(-1).tolist()
    excused = []
    for r in bad:
        assert not greedy[r] and int(mode[r]) not in (0, 2), f"row {r} (mode {int(mode[r])}): kernel {int(ids[r])}, reference {int(ref[r])}"
        two = race[r].topk(2).values.double()
        near_race = bool((two[0] - two[1]).abs() <= 1e-6 * two.abs().max())
        near_p = bool(p_on[r]) and bool(((mass[r] - float(prm[2][r])).abs() < 1e-5).any())
        assert near_race or near_p, f"row {r}: kernel {int(ids[r])}, reference {int(ref[r])}, no tie within the tolerances"
        excused.append(r)
    return excused


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
@pytest.mark.parametrize("vocab", VOCABS)
def test_kernel_matches_reference(dtype, vocab):
    g = torch.Generator().manual_seed(vocab)
    rows = 40
    mode, prm = _mixed_params(rows, g)
    x = (torch.randn(rows, vocab, generator=g) * 3).to(dtype)
    x[1, 5:9] = x[1].max()                              # ties at the top
    excused = _compare(x.cuda(), prm, mode)
    if excused:
        print(f"excused rows (boundary or race ties): {excused}")
    assert len(excused) <= 2


@pytest.mark.parametrize("rows", [1, 7, 131, 512])
def test_row_counts_and_strided_rows(rows):
    g = torch.Generator().manual_seed(rows)
    mode, prm = _mixed_params(rows, g)
    big = (torch.randn(rows, 32000 + 96, generator=g) * 2).to(torch.bfloat16).cuda()
    x = big[:, 3:32003]                                  # row stride 32096, rows not 16-byte aligned
    assert x.stride(0) == 32096 and (rows == 1 or not x.is_contiguous())
    excused = _compare(x, prm, mode)
    assert len(excused) <= max(2, rows // 50)


def test_probabilities_threshold_and_return_top():
    g = torch.Generator().manual_seed(5)
    rows, vocab = 64, 32000
    p = torch.softmax(torch.randn(rows, vocab, generator=g) * 4, -1)
    mode, prm = _mixed_params(rows, g)
    prm[0] = torch.ones(rows)
    mode = torch.full((rows,), 3)
    thr = torch.rand(rows, generator=g) * 0.05
    for truncated in (True, False):
        assert len(_compare(p.cuda(), prm, mode, threshold=thr, is_prob=True, truncated=truncated)) <= 2
    got = sampling.sample(p.cuda(), *[q.cuda() for q in prm], is_prob=True, k_out=50)
    ref = torch.topk(p, 50)
    assert torch.equal(got[2].cpu(), ref.values) and torch.equal(got[3].cpu(), ref.indices)


def test_fp16_adjacent_values_select_exactly():
    """16 adjacent fp16 values (1 + j * 2^-10) share their top 16 key bits in groups of 8: the top-k and top-p cutoffs must still
    fall between neighbouring values, not at bucket granularity."""
    g = torch.Generator().manual_seed(11)
    rows, vocab = 256, 4096
    row = -4 * torch.rand(vocab, generator=g)
    pos = torch.randperm(vocab, generator=g)[:16]
    row[pos] = 1 + torch.arange(16) * 2.0 ** -10
    x = row.half().reshape(1, -1).expand(rows, -1).contiguous()
    order = pos.flip(0)                                   # positions of the largest, second largest, ... planted values
    mode = torch.tensor([2, 2, 3, 4]).repeat(rows // 4)
    top_k = torch.tensor([1, 3, 0, 10]).repeat(rows // 4).int()
    top_p = torch.tensor([1.0, 1.0, 0.3, 0.3]).repeat(rows // 4)
    prm = [torch.full((rows,), 0.05), top_k, top_p, torch.arange(rows) * 104729, torch.zeros(rows, dtype=torch.int64)]
    assert _compare(x.cuda(), prm, mode) == []
    ids = sampling.sample(x.cuda(), *[q.cuda() for q in prm])[0].cpu()
    assert (ids[0::4] == order[0]).all()
    assert set(ids[1::4].tolist()) <= set(order[:3].tolist())
    kept = set(order[:5].tolist())                        # about 1/16 of the mass each: top_p = 0.3 keeps the five largest
    assert set(ids[2::4].tolist()) <= kept and set(ids[3::4].tolist()) <= kept


@pytest.mark.parametrize("dtype", DTYPES, ids=str)
def test_return_top_with_ties_and_negative_values(dtype):
    """k near 1024 over rows full of ties (a flat fp16 distribution, logits of few distinct negative values) against the reference's
    stable descending order."""
    g = torch.Generator().manual_seed(13)
    rows, vocab, k = 4, 8192, 1000
    flat = ((1 + 0.01 * torch.rand(rows, vocab, generator=g)) / vocab).to(dtype)
    neg = (-torch.randint(1, 40, (rows, vocab), generator=g).float() / 8).to(dtype)
    prm = [torch.ones(rows), torch.zeros(rows, dtype=torch.int32), torch.ones(rows), torch.arange(rows), torch.zeros(rows, dtype=torch.int64)]
    for x, is_prob in ((flat, True), (neg, False)):
        got = sampling.sample(x.cuda(), *[q.cuda() for q in prm], is_prob=is_prob, k_out=k)
        want = sampling.sample_ref(x, *prm, is_prob=is_prob, k_out=k)
        assert torch.equal(got[2].cpu(), want[2]) and torch.equal(got[3].cpu(), want[3])
        assert torch.equal(got[2].cpu(), torch.topk(x.float(), k).values.to(dtype))
    with pytest.raises(RuntimeError):
        ext().sample_tokens(flat[:, :16].cuda(), *[q.cuda() for q in prm[:3]], None, *[q.cuda() for q in prm[3:]], True, True, 17)


def test_sampling_call_does_not_synchronize():
    g = torch.Generator().manual_seed(3)
    mode, prm = _mixed_params(8, g)
    x = torch.randn(8, 1000, generator=g).cuda()
    prm = [q.cuda() for q in prm]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        sampling.sample(x, *prm, k_out=4)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_philox_draws_match_the_reference():
    like = torch.empty(1, device="cuda")
    for seed, off in ((0, 0), (2 ** 63 - 1, 2 ** 40 + 3), (-5, 17)):
        assert torch.equal(ext().sampling_uniforms(seed, off, 4099, like).cpu(), sampling.uniforms(seed, off, 4099))


def test_top_p_sampling_cuda_equals_cpu():
    g = torch.Generator().manual_seed(9)
    p = torch.softmax(torch.randn(16, 5000, generator=g) * 3, -1)
    ps = torch.rand(16, generator=g) * 0.9 + 0.05
    seeds = torch.randint(0, 2 ** 40, (16,), generator=g)
    thr = torch.full((16,), 1e-3)
    for mode in ("truncated", "non-truncated"):
        cpu = paddle.top_p_sampling(p, ps, threshold=thr, topp_seed=seeds, k=8, mode=mode, return_top=True)
        gpu = paddle.top_p_sampling(p.cuda(), ps.cuda(), threshold=thr.cuda(), topp_seed=seeds.cuda(), k=8, mode=mode, return_top=True)
        for a, b in zip(cpu, gpu):
            assert torch.equal(torch.as_tensor(a), torch.as_tensor(b).cpu())


def _gpu_model(seed=0):
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(seed)
        cfg = models.llama_tiny(hidden_size=256, intermediate_size=512, num_attention_heads=2, num_key_value_heads=2, num_hidden_layers=2,
                                vocab_size=32000)
        m = models.LlamaForCausalLM(cfg)
        m.eval()
    finally:
        paddle.set_default_dtype("float32")
    return m, cfg


def test_engine_greedy_and_seeded_requests():
    m, cfg = _gpu_model()
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, cfg.vocab_size, (int(n),), generator=g).tolist() for n in torch.randint(3, 20, (32,), generator=g)]
    greedy = [models.generate(m, torch.tensor([p], device="cuda"), max_new_tokens=8).as_subclass(torch.Tensor)[0, len(p):].tolist()
              for p in prompts[3:7]]
    kw = dict(do_sample=True, temperature=0.9, top_k=40, top_p=0.9)

    def alone(p, seed):
        eng = models.LLMEngine(m, num_blocks=64, block_size=16)
        i = eng.add_request(p, 8, seed=seed, **kw)
        return eng.run_until_done()[i]

    want = [alone(p, 100 + j) for j, p in enumerate(prompts[:3])]
    eng = models.LLMEngine(m, num_blocks=256, block_size=16)
    ids = [eng.add_request(p, 8, seed=100 + j, **kw) if j < 3 else eng.add_request(p, 8) if j < 7 else eng.add_request(p, 8, **kw)
           for j, p in enumerate(prompts)]
    res = eng.run_until_done()
    assert [res[i] for i in ids[:3]] == want
    assert [res[i] for i in ids[3:7]] == greedy
    eng = models.LLMEngine(m, num_blocks=5, block_size=16)            # too few blocks for everyone: preemption
    ids = [eng.add_request(p + [7] * 20, 8, seed=300 + j, **kw) for j, p in enumerate(prompts[:3])]
    res = eng.run_until_done()
    assert eng.stats["preemptions"] >= 1
    assert [res[i] for i in ids] == [alone(p + [7] * 20, 300 + j) for j, p in enumerate(prompts[:3])]
