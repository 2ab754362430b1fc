"""head_dim 64 on the paged attention kernels (decode, verify rows and prefill behind block_attention, contiguous decode behind
generate()), against the reference in mixed batches, verify rows against successive decode, which batches still take the reference, and
LLMEngine on 64-wide-head models, alone and as a speculative draft (needs a GPU)."""
import math

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import kernels, models
from paddle_b200.framework.flags import set_flags
from paddle_b200.incubate.nn import paged_attention as PA

pytestmark = pytest.mark.gpu

D = 64


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _ext():
    from paddle_b200._build import ext

    return ext()


def _raw(t):
    return t.as_subclass(torch.Tensor)


def _batch(specs, nh, nkv, bs, dtype, seed=0):
    """specs: [(enc, dec, now)].  Shuffled block tables; every cache row that holds no cached token is NaN, and so are the blocks that
    table entries past a sequence's own blocks point at."""
    g = torch.Generator().manual_seed(seed)
    now = torch.tensor([s[2] for s in specs], dtype=torch.int32)
    cu = torch.zeros(len(specs) + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(now, 0)
    need = [((0 if e > 0 else d) + n + bs - 1) // bs for e, d, n in specs]
    max_blocks, nblocks = max(need) + 2, sum(need) + 8
    perm = torch.randperm(nblocks, generator=g)
    spare = perm[sum(need):]
    bt = spare[torch.randint(0, spare.numel(), (len(specs), max_blocks), generator=g)].to(torch.int32)
    kc = torch.full((nblocks, nkv, bs, D), float("nan"), dtype=dtype)
    vc = torch.full_like(kc, float("nan"))
    nxt = 0
    for b, (e, d, n) in enumerate(specs):
        bt[b, :need[b]] = perm[nxt:nxt + need[b]].to(torch.int32)
        nxt += need[b]
        pos = torch.arange(0 if e > 0 else d)                    # the cached prefix; everything else stays NaN
        blk = bt[b].long()[pos // bs]
        kc[blk, :, pos % bs] = (torch.randn(pos.numel(), nkv, D, generator=g) * 0.5).to(dtype)
        vc[blk, :, pos % bs] = (torch.randn(pos.numel(), nkv, D, generator=g) * 0.5).to(dtype)
    qkv = (torch.randn(int(cu[-1]), (nh + 2 * nkv) * D, generator=g) * 0.5).to(dtype)
    enc = torch.tensor([s[0] for s in specs], dtype=torch.int32)
    dec = torch.tensor([s[1] for s in specs], dtype=torch.int32)
    args = (enc.cuda(), dec.cuda(), now.cuda(), cu.cuda(), bt.cuda(), bs)
    return qkv.cuda(), kc.cuda(), vc.cuda(), args


# decode rows, fresh prompts, continuing chunks, verify rows of 2 .. VERIFY_MAX tokens (those over the 64-row tile go to prefill) and
# zero-length rows
SPECS = ([(0, 7, 1), (37, 0, 37), (0, 50, 0), (300, 0, 300), (0, 129, 200), (0, 1000, 1), (0, 64, 0)]
         + [(0, past, now) for past in (1, 63, 64, 1000) for now in range(2, PA.VERIFY_MAX + 1, 3)] + [(0, 300, 1)])


@pytest.mark.parametrize("heads", [(32, 4), (8, 8), (16, 2)])
@pytest.mark.parametrize("bs", [16, 32, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_mixed_batch_matches_reference(dtype, bs, heads):
    nh, nkv = heads
    qkv, kc0, vc0, args = _batch(SPECS, nh, nkv, bs, dtype)
    kernels.reset_launch_count()
    out, _, kc1, vc1 = PA.block_attention(qkv, kc0.clone(), vc0.clone(), *args)
    assert kernels.launch_count() >= 6                           # decode, verify and prefill: two launches each
    ref, _, kc2, vc2 = PA._block_attention_ref(qkv, kc0.clone(), vc0.clone(), *args)
    assert torch.equal(_raw(kc1).nan_to_num(7.0), _raw(kc2).nan_to_num(7.0)) and torch.equal(_raw(vc1).nan_to_num(7.0), _raw(vc2).nan_to_num(7.0))
    o, r = _raw(out).float(), _raw(ref).float()
    assert torch.isfinite(o).all()
    cu = args[3].tolist()
    for b in range(len(SPECS)):
        e = rel_err(o[cu[b]:cu[b + 1]], r[cu[b]:cu[b + 1]]) if cu[b + 1] > cu[b] else 0.0
        assert e < 2e-2, (b, SPECS[b], e)


@pytest.mark.parametrize("past,n", [(1, 2), (63, 5), (1000, 8), (6000, 16)])
def test_verify_row_equals_successive_decode(past, n):
    g = torch.Generator(device="cuda").manual_seed(past)
    nh, nkv, bs = 8, 2, 64
    total = past + n
    nblk = (total + bs - 1) // bs
    perm = torch.randperm(nblk + 6, device="cuda", generator=g)
    bt = torch.cat([perm[:nblk], perm[nblk:nblk + 2]]).to(torch.int32).reshape(1, -1).contiguous()   # two NaN blocks past the end
    kc = torch.full((nblk + 6, nkv, bs, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    vc = torch.full_like(kc, float("nan"))
    pos = torch.arange(total, device="cuda")
    blk = bt[0].long()[pos // bs]
    kc[blk, :, pos % bs] = (torch.randn(total, nkv, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    vc[blk, :, pos % bs] = (torch.randn(total, nkv, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    q = (torch.randn(n, nh, D, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    scale = 1.0 / math.sqrt(D)
    out = torch.zeros(n, nh * D, device="cuda", dtype=torch.bfloat16)
    _ext().decode_attention_paged_multi(q, kc, vc, bt, i32(0), i32(n), i32(past), scale, out)
    assert torch.isfinite(out.float()).all()
    for j in range(n):
        one = _ext().decode_attention_paged(q[j:j + 1].contiguous(), kc, vc, i32(past + j + 1), bt, scale)
        assert rel_err(out[j], one.reshape(-1)) < 2e-2, j


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_contiguous_decode_matches_fp32_reference(dtype):
    g = torch.Generator(device="cuda").manual_seed(3)
    b, nh, nkv, smax = 5, 16, 4, 3000
    lens = torch.tensor([1, 17, 256, 2999, 3000], dtype=torch.int32, device="cuda")
    q = torch.randn(b, nh, D, device="cuda", generator=g).to(dtype)
    kc = torch.randn(b, nkv, smax, D, device="cuda", generator=g).to(dtype)
    vc = torch.randn(b, nkv, smax, D, device="cuda", generator=g).to(dtype)
    for i, n in enumerate(lens.tolist()):                        # positions past lens[b] are never read
        kc[i, :, n:] = float("nan")
        vc[i, :, n:] = float("nan")
    scale = 1.0 / math.sqrt(D)
    out = _ext().decode_attention(q, kc, vc, lens, scale)
    for i, n in enumerate(lens.tolist()):
        k = kc[i, :, :n].float().repeat_interleave(nh // nkv, 0)
        v = vc[i, :, :n].float().repeat_interleave(nh // nkv, 0)
        ref = torch.einsum("hs,hsd->hd", torch.softmax(torch.einsum("hd,hsd->hs", q[i].float(), k) * scale, -1), v)
        assert rel_err(out[i], ref) < 1e-2, (i, n)


def _llama(**kw):
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        base = dict(hidden_size=512, intermediate_size=1024, num_attention_heads=8, num_key_value_heads=2, num_hidden_layers=2, vocab_size=512,
                    max_position_embeddings=1024)
        base.update(kw)
        cfg = models.llama_tiny(**base)
        return models.LlamaForCausalLM(cfg), cfg
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")


def _assert_same_greedy(m, prompt, got, want):
    """Two greedy continuations of `prompt` through different attention paths are equal, or part at a near-tie: where they first differ,
    the full forward over prompt + the common tokens scores the two picks within 2 % of its largest logit."""
    assert len(got) == len(want)
    i = next((j for j in range(len(want)) if got[j] != want[j]), None)
    if i is None:
        return
    ids = torch.tensor([prompt + want[:i]], device="cuda")
    with torch.no_grad():
        logits = _raw(m(ids.as_subclass(paddle.Tensor))).float()[0, -1]
    assert (logits[want[i]] - logits[got[i]]).abs() < 0.02 * logits.abs().max(), (i, got, want)


def test_generate_decode_kernel_matches_masked_softmax(monkeypatch):
    m, cfg = _llama()
    assert m.llama.layers[0].self_attn.head_dim == D
    g = torch.Generator().manual_seed(1)
    prompt = torch.randint(1, cfg.vocab_size, (150,), generator=g).tolist()
    calls = []
    dec = _ext().decode_attention
    monkeypatch.setattr(_ext(), "decode_attention", lambda *a: calls.append(1) or dec(*a))
    outs = []
    for on in (False, True):
        set_flags({"FLAGS_b200_decode_kernel": on})
        try:
            out = models.generate(m, torch.tensor([prompt], device="cuda"), max_new_tokens=12).as_subclass(torch.Tensor)
        finally:
            set_flags({"FLAGS_b200_decode_kernel": False})
        outs.append(out[0, len(prompt):].tolist())
        assert bool(calls) == on
    _assert_same_greedy(m, prompt, outs[1], outs[0])


def _no_reference(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("head_dim 64 batch reached _block_attention_ref")

    monkeypatch.setattr(PA, "_block_attention_ref", boom)


def test_16bit_batches_never_call_the_reference_and_the_rest_still_do(monkeypatch):
    qkv, kc, vc, args = _batch(SPECS, 8, 2, 64, torch.bfloat16, seed=4)
    ref = PA._block_attention_ref
    calls = []
    monkeypatch.setattr(PA, "_block_attention_ref", lambda *a, **k: calls.append(1) or ref(*a, **k))
    out = PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args)[0]
    assert not calls and torch.isfinite(_raw(out).float()).all()
    nkv = kc.shape[1]
    ones = torch.ones(nkv, device="cuda")
    k8, v8 = torch.zeros(kc.shape, dtype=torch.int8, device="cuda"), torch.zeros(vc.shape, dtype=torch.int8, device="cuda")
    PA.block_attention(qkv.clone(), k8, v8, *args, cache_k_quant_scales=ones, cache_v_quant_scales=ones, cache_k_dequant_scales=ones,
                       cache_v_dequant_scales=ones)
    assert len(calls) == 1
    rope = torch.randn(2, 1, 2048, 1, D // 2, device="cuda")
    PA.block_attention(qkv.clone(), kc.clone(), vc.clone(), *args, rope_emb=rope)
    assert len(calls) == 2


@pytest.mark.parametrize("mode", ["whole", "chunked", "prefix_caching"])
def test_engine_on_a_64d_model_matches_generate(monkeypatch, mode):
    m, cfg = _llama()
    g = torch.Generator().manual_seed(2)
    system = torch.randint(1, cfg.vocab_size, (160,), generator=g).tolist()
    prompts = [system + torch.randint(1, cfg.vocab_size, (k,), generator=g).tolist() for k in (5, 40, 17)]
    n = 12
    want = [models.generate(m, torch.tensor([p], device="cuda"), max_new_tokens=n).as_subclass(torch.Tensor)[0, len(p):].tolist()
            for p in prompts]
    _no_reference(monkeypatch)
    kw = {"chunked": dict(max_prefill_chunk=48), "prefix_caching": dict(enable_prefix_caching=True)}.get(mode, {})
    eng = models.LLMEngine(m, num_blocks=128, block_size=16, **kw)
    ids = [eng.add_request(prompts[0], n)]
    eng.step()                                                   # later requests find the first one's blocks when caching
    ids += [eng.add_request(p, n) for p in prompts[1:]]
    got = eng.run_until_done()
    for i, p, w in zip(ids, prompts, want):
        _assert_same_greedy(m, p, got[i], w)


def test_speculative_engine_with_a_64d_draft_matches_the_target_alone(monkeypatch):
    target, cfg = _llama(num_attention_heads=4, num_key_value_heads=2)        # head_dim 128
    draft, _ = _llama(hidden_size=256, intermediate_size=512, num_attention_heads=4, num_key_value_heads=2)   # head_dim 64
    assert target.llama.layers[0].self_attn.head_dim == 128 and draft.llama.layers[0].self_attn.head_dim == D
    g = torch.Generator().manual_seed(5)
    prompts = [torch.randint(1, cfg.vocab_size, (k,), generator=g).tolist() for k in (30, 200)]
    n = 16
    plain = models.LLMEngine(target, num_blocks=128, block_size=16)
    ids = [plain.add_request(p, n) for p in prompts]
    want = plain.run_until_done()
    _no_reference(monkeypatch)
    spec = models.LLMEngine(target, num_blocks=128, block_size=16, draft_model=draft, num_speculative_tokens=4)
    draft_rows = []
    run = spec._run
    spec._run = lambda net, seqs, n_new, *a, **k: (draft_rows.append(sum(n_new)) if net is not spec._target else None) or run(net, seqs, n_new, *a, **k)
    sids = [spec.add_request(p, n) for p in prompts]
    got = spec.run_until_done()
    assert draft_rows                                            # the draft ran, on the kernels
    for i, j, p in zip(ids, sids, prompts):
        _assert_same_greedy(target, p, got[j], want[i])
