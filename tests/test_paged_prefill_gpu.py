"""Prefill attention over the paged KV cache (csrc/attention_sm100.cu, PAGED instantiation, behind incubate.nn.paged_attention.block_attention)
against the per-token reference, against the dense kernel bit for bit, and end to end through LLMEngine chunked prefill (needs a GPU)."""
import math

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import kernels, models
from paddle_b200.incubate.nn import paged_attention as PA

pytestmark = pytest.mark.gpu

D = 128


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _ext():
    from paddle_b200._build import ext

    return ext()


def _batch(specs, nh, nkv, bs, dtype, seed=0):
    """specs: [(enc, dec, now)].  Shuffled block tables; every cache row that holds no token of a sequence is NaN, and so is every
    table entry past a sequence's blocks' worth of pool (the tables point at NaN blocks there)."""
    g = torch.Generator().manual_seed(seed)
    enc = torch.tensor([s[0] for s in specs], dtype=torch.int32)
    dec = torch.tensor([s[1] for s in specs], dtype=torch.int32)
    now = torch.tensor([s[2] for s in specs], dtype=torch.int32)
    cu = torch.zeros(len(specs) + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(now, 0)
    need = [((0 if e > 0 else d) + n + bs - 1) // bs for e, d, n in specs]
    max_blocks = max(need) + 2
    nblocks = sum(need) + 8
    perm = torch.randperm(nblocks, generator=g)
    spare = perm[sum(need):]
    bt = spare[torch.randint(0, spare.numel(), (len(specs), max_blocks), generator=g)].to(torch.int32)   # unused entries: NaN blocks
    kc = torch.full((nblocks, nkv, bs, D), float("nan"), dtype=dtype)
    vc = torch.full((nblocks, nkv, bs, D), float("nan"), dtype=dtype)
    nxt = 0
    for b, (e, d, n) in enumerate(specs):
        bt[b, :need[b]] = perm[nxt:nxt + need[b]].to(torch.int32)
        nxt += need[b]
        past = 0 if e > 0 else d
        for pos in range(past):                                  # the cached prefix; everything else stays NaN
            blk, off = int(bt[b, pos // bs]), pos % bs
            kc[blk, :, off] = (torch.randn(nkv, D, generator=g) * 0.5).to(dtype)
            vc[blk, :, off] = (torch.randn(nkv, D, generator=g) * 0.5).to(dtype)
    qkv = (torch.randn(int(cu[-1]), (nh + 2 * nkv) * D, generator=g) * 0.5).to(dtype)
    args = (enc.cuda(), dec.cuda(), now.cuda(), cu.cuda(), bt.cuda(), bs)
    return qkv.cuda(), kc.cuda(), vc.cuda(), args


# decode rows, fresh prompts and continuing chunks with past in {5, 127, 128, 1000} and now in {2, 129, 300}
SPECS = ([(0, 7, 1), (37, 0, 37), (0, 300, 1), (300, 0, 300)]
         + [(0, past, now) for past in (5, 127, 128, 1000) for now in (2, 129, 300)] + [(0, 64, 1)])


@pytest.mark.parametrize("heads", [(8, 2), (4, 4)])
@pytest.mark.parametrize("bs", [16, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_block_attention_mixed_batch_matches_reference(dtype, bs, heads):
    nh, nkv = heads
    qkv, kc0, vc0, args = _batch(SPECS, nh, nkv, bs, dtype)
    kernels.reset_launch_count()
    out, _, kc1, vc1 = PA.block_attention(qkv, kc0.clone(), vc0.clone(), *args)
    assert kernels.launch_count() >= 4                           # paged decode (2 launches) + work list and paged prefill
    ref, _, kc2, vc2 = PA._block_attention_ref(qkv, kc0.clone(), vc0.clone(), *args)
    raw = lambda t: t.as_subclass(torch.Tensor)                  # noqa: E731
    assert torch.equal(raw(kc1).nan_to_num(7.0), raw(kc2).nan_to_num(7.0)) and torch.equal(raw(vc1).nan_to_num(7.0), raw(vc2).nan_to_num(7.0))
    o, r = raw(out).float(), raw(ref).float()
    assert torch.isfinite(o).all()
    cu = args[3].tolist()
    for b in range(len(SPECS)):
        assert rel_err(o[cu[b]:cu[b + 1]], r[cu[b]:cu[b + 1]]) < 2e-2, (b, SPECS[b])


def test_cuda_path_never_calls_the_reference(monkeypatch):
    qkv, kc, vc, args = _batch(SPECS, 8, 2, 64, torch.bfloat16, seed=1)

    def boom(*a, **k):
        raise AssertionError("reference called on the CUDA path")

    monkeypatch.setattr(PA, "_block_attention_ref", boom)
    out, _, _, _ = PA.block_attention(qkv, kc, vc, *args)
    assert torch.isfinite(out.as_subclass(torch.Tensor).float()).all()


@pytest.mark.parametrize("bs", [16, 64, 256])
def test_paged_prefill_is_bitwise_the_dense_kernel(bs):
    """2048 new rows over a 6000-token prefix: the same tiles and the same arithmetic as attention_fwd on the gathered K / V."""
    torch.manual_seed(0)
    nh, nkv, past, n = 8, 2, 6000, 2048
    total = past + n
    nblk = (total + bs - 1) // bs
    pool = nblk + 5
    perm = torch.randperm(pool, device="cuda")
    bt = perm[:nblk].to(torch.int32).reshape(1, -1).contiguous()
    kc = torch.full((pool, nkv, bs, D), float("nan"), device="cuda", dtype=torch.bfloat16)
    vc = torch.full_like(kc, float("nan"))
    K = (torch.randn(total, nkv, D, device="cuda") * 0.5).to(torch.bfloat16)
    V = (torch.randn(total, nkv, D, device="cuda") * 0.5).to(torch.bfloat16)
    pos = torch.arange(total, device="cuda")
    kc[bt[0].long()[pos // bs], :, pos % bs] = K
    vc[bt[0].long()[pos // bs], :, pos % bs] = V
    q = (torch.randn(n, nh, D, device="cuda") * 0.5).to(torch.bfloat16)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    out = torch.zeros(n, nh * D, device="cuda", dtype=torch.bfloat16)
    lse = torch.zeros(nh, n, device="cuda", dtype=torch.float32)
    scale = 1.0 / math.sqrt(D)
    _ext().attention_fwd_paged(q, kc, vc, bt, i32(0), i32(n), i32(past), scale, out, lse)
    ref, ref_lse = _ext().attention_fwd(q.unsqueeze(0), K.unsqueeze(0), V.unsqueeze(0), scale, True)
    assert torch.isfinite(out.float()).all()
    assert torch.equal(out, ref.reshape(n, nh * D))
    assert torch.equal(lse, ref_lse[0])


def test_engine_chunked_prefill_logits_match_whole_prefill():
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.llama_tiny(hidden_size=256, intermediate_size=512, num_attention_heads=2, num_key_value_heads=2, num_hidden_layers=2,
                                vocab_size=512, max_position_embeddings=1024)
        m = models.LlamaForCausalLM(cfg)
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    g = torch.Generator().manual_seed(0)
    prompt = torch.randint(1, cfg.vocab_size, (300,), generator=g).tolist()
    logits = {}
    for chunk in (None, 128):
        eng = models.LLMEngine(m, num_blocks=64, block_size=16, max_prefill_chunk=chunk)
        assert eng.device.type == "cuda" and eng.hd == D
        calls = []
        fwd = eng._forward
        eng._forward = lambda *a, _f=fwd, _c=calls: _c.append(_f(*a)) or _c[-1]
        eng.add_request(prompt, 2)
        eng.run_until_done()
        logits[chunk] = calls[0 if chunk is None else 2][0].float()   # the forward that ends the prompt (3 chunks: 128, 128, 44)
    assert torch.isfinite(logits[128]).all()
    assert rel_err(logits[128], logits[None]) < 2e-2
