"""Shared-prefix decode (csrc/decode_attention.cu, `decode_attention_paged_shared`, behind block_attention's shared_prefix groups) against
the reference in mixed batches, its 8-bit instantiations bit for bit against the 16-bit one, NaN rows for members that break the group
contract, and LLMEngine prefix caching against an engine without it (needs a GPU)."""
import math
import os
import re
import subprocess

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import kernels, models
from paddle_b200.incubate.nn import paged_attention as PA
from test_kv_cache_quant_gpu import _pow2_scales, _random_8bit
from test_paged_prefill_gpu import _ext, rel_err

pytestmark = pytest.mark.gpu

D = 128


def _shared_batch(groups, others, nh, nkv, bs, dtype, seed=0):
    """groups: [(prefix_len, [suffix per member])]; a member brings one new token and has prefix_len + suffix - 1 cached ones, its first
    prefix_len / bs blocks shared with its group.  others: [(enc, dec, now)] rows outside the groups.  Shuffled block tables; every cache
    row that holds no cached token is NaN, and so is every block a table names past a sequence's end."""
    g = torch.Generator().manual_seed(seed)
    rows, tables, shared = [], [], []                  # rows: (enc, dec, now)
    nxt = 0
    for plen, sufs in groups:
        pre = list(range(nxt, nxt + plen // bs))
        nxt += plen // bs
        cu_m = len(rows)
        for suf in sufs:
            past = plen + suf - 1
            own = (past + 1 + bs - 1) // bs - plen // bs
            tables.append(pre + list(range(nxt, nxt + own)))
            nxt += own
            rows.append((0, past, 1))
        shared.append((cu_m, len(rows), plen))
    for e, d, n in others:
        k = ((0 if e > 0 else d) + n + bs - 1) // bs
        tables.append(list(range(nxt, nxt + k)))
        nxt += k
        rows.append((e, d, n))
    nblocks = nxt + 6
    perm = torch.randperm(nblocks, generator=g)
    max_blocks = max(len(t) for t in tables) + 2
    bt = perm[nxt + torch.randint(0, 6, (len(rows), max_blocks), generator=g)]          # unused entries: NaN blocks
    for i, t in enumerate(tables):
        bt[i, :len(t)] = perm[torch.tensor(t, dtype=torch.long)]
    bt = bt.to(torch.int32)
    kc = torch.full((nblocks, nkv, bs, D), float("nan"), dtype=dtype)
    vc = torch.full_like(kc, float("nan"))
    written = torch.zeros(nblocks, bs, dtype=torch.bool)
    for i, (e, d, n) in enumerate(rows):
        past = 0 if e > 0 else d
        pos = torch.arange(past)
        blk, off = bt[i].long()[pos // bs], pos % bs
        new = ~written[blk, off]                       # a shared row is written once
        blk, off = blk[new], off[new]
        written[blk, off] = True
        kc[blk, :, off] = (torch.randn(blk.numel(), nkv, D, generator=g) * 0.5).to(dtype)
        vc[blk, :, off] = (torch.randn(blk.numel(), nkv, D, generator=g) * 0.5).to(dtype)
    now = torch.tensor([r[2] for r in rows], dtype=torch.int32)
    cu = torch.zeros(len(rows) + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(now, 0)
    qkv = (torch.randn(int(cu[-1]), (nh + 2 * nkv) * D, generator=g) * 0.5).to(dtype)
    enc = torch.tensor([r[0] for r in rows], dtype=torch.int32)
    dec = torch.tensor([r[1] for r in rows], dtype=torch.int32)
    sp = ([0] + [b for _, b, _ in shared], list(range(shared[-1][1])), [p for _, _, p in shared])   # members: batch 0 .. n-1, by group
    return qkv.cuda(), kc.cuda(), vc.cuda(), (enc.cuda(), dec.cuda(), now.cuda(), cu.cuda(), bt.cuda(), bs), sp


def _groups(bs, g):
    """Group sizes 1, 2, 7 and 40; prefixes from one block to about 6,000 tokens; suffixes 1 .. 300."""
    suf = lambda n: torch.randint(1, 301, (n,), generator=g).tolist()     # noqa: E731
    return [(bs, [1]), ((6000 // bs) * bs, [300, 1]), ((1000 // bs) * bs, suf(6) + [64]), ((2048 // bs) * bs, suf(38) + [1, 300])]


OTHERS = [(0, 7, 1), (0, 1000, 1), (0, 63, 4), (300, 0, 300), (0, 129, 200)]     # decode rows, a verify row, prefill rows


@pytest.mark.parametrize("heads", [(32, 8), (8, 2), (4, 4), (32, 32), (32, 4)])
@pytest.mark.parametrize("bs", [16, 64, 256])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_grouped_decode_rows_in_mixed_batches_match_reference(dtype, bs, heads):
    nh, nkv = heads
    g = torch.Generator().manual_seed(bs + nh)
    qkv, kc0, vc0, args, sp = _shared_batch(_groups(bs, g), OTHERS, nh, nkv, bs, dtype, seed=bs)
    out, _, kc1, vc1 = PA.block_attention(qkv, kc0.clone(), vc0.clone(), *args, shared_prefix=sp)
    ref, _, kc2, vc2 = PA._block_attention_ref(qkv, kc0.clone(), vc0.clone(), *args, shared_prefix=sp)
    raw = lambda t: t.as_subclass(torch.Tensor)                  # noqa: E731
    assert torch.equal(raw(kc1).nan_to_num(7.0), raw(kc2).nan_to_num(7.0)) and torch.equal(raw(vc1).nan_to_num(7.0), raw(vc2).nan_to_num(7.0))
    o, r = raw(out).float(), raw(ref).float()
    assert torch.isfinite(o).all()
    cu = args[3].tolist()
    for b in range(len(cu) - 1):
        e = rel_err(o[cu[b]:cu[b + 1]], r[cu[b]:cu[b + 1]])
        assert e < 2e-2, (b, e)


def _direct(nh, nkv, bs, dtype, groups, seed):
    """Operands of a direct decode_attention_paged_shared call: only grouped decode rows (q [n, H, D], one row per member)."""
    qkv, kc, vc, args, sp = _shared_batch(groups, [], nh, nkv, bs, dtype, seed=seed)
    enc, dec, now, cu, bt, _ = args
    q = qkv.reshape(qkv.shape[0], nh + 2 * nkv, D)[:, :nh]
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)          # noqa: E731
    return q, kc, vc, bt, cu[:-1].contiguous(), (dec + 1).contiguous(), tuple(i32(v) for v in sp)


@pytest.mark.parametrize("kv", [torch.int8, torch.float8_e4m3fn])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_quantized_shared_decode_is_bitwise_the_16bit_kernel(dtype, kv):
    nh, nkv, bs = 8, 2, 16
    q, kc, vc, bt, cu, lens, sp = _direct(nh, nkv, bs, dtype, [(992, [5, 77, 300]), (16, [1, 40]), (4096, [33] * 40)], seed=3)
    g = torch.Generator(device="cuda").manual_seed(1)
    kc8, vc8 = _random_8bit(tuple(kc.shape), kv, g), _random_8bit(tuple(vc.shape), kv, g)
    kdq, vdq = _pow2_scales(nkv, 5), _pow2_scales(nkv, 6)
    kc16 = (kc8.float() * kdq[None, :, None, None]).to(dtype)
    vc16 = (vc8.float() * vdq[None, :, None, None]).to(dtype)
    scale = 1.0 / math.sqrt(D)
    outs = []
    for k, v, dq in ((kc8, vc8, dict(k_dequant_scales=kdq, v_dequant_scales=vdq)), (kc16, vc16, {})):
        out = torch.zeros(q.shape[0], nh * D, device="cuda", dtype=dtype)
        _ext().decode_attention_paged_shared(q, k, v, bt, cu, lens, *sp, scale, out, **dq)
        outs.append(out)
    assert torch.isfinite(outs[0].float()).all()
    assert torch.equal(outs[0], outs[1])


def test_members_breaking_the_contract_get_nan_rows():
    nh, nkv, bs = 8, 2, 64
    q, kc, vc, bt, cu, lens, sp = _direct(nh, nkv, bs, torch.bfloat16, [(1024, [5, 9, 70, 3])], seed=4)
    scale = 1.0 / math.sqrt(D)
    good = _ext().decode_attention_paged(q.contiguous(), kc, vc, lens, bt, scale).reshape(q.shape[0], nh * D)
    bt_bad = bt.clone()
    bt_bad[1, 3] = bt[1, -1]                                   # member 1's fourth prefix block is another block
    lens_bad = lens.clone()
    lens_bad[3] = 1024                                         # member 3 has only 1023 cached tokens: the 1024-token prefix is too long
    out = torch.zeros(q.shape[0], nh * D, device="cuda", dtype=torch.bfloat16)
    _ext().decode_attention_paged_shared(q, kc, vc, bt_bad, cu, lens_bad, *sp, scale, out)
    assert torch.isnan(out[1].float()).all() and torch.isnan(out[3].float()).all()
    for i in (0, 2):
        assert rel_err(out[i], good[i]) < 2e-2, i
    with pytest.raises(RuntimeError):                          # the binding checks what the host can see
        _ext().decode_attention_paged_shared(q, kc, vc, bt, cu, lens, sp[0], torch.tensor([0, 1, 1, 2], dtype=torch.int32), sp[2], scale, out)
    with pytest.raises(RuntimeError):
        _ext().decode_attention_paged_shared(q, kc, vc, bt, cu, lens, sp[0], sp[1], torch.tensor([1000], dtype=torch.int32), scale, out)


def test_all_grouped_rows_skip_the_decode_kernel(monkeypatch):
    nh, nkv, bs = 32, 8, 64
    qkv, kc, vc, args, sp = _shared_batch([(2048, [64] * 16), (1024, [3, 200])], [], nh, nkv, bs, torch.bfloat16, seed=5)

    def boom(*a, **k):
        raise AssertionError("unexpected call on the grouped-decode path")

    monkeypatch.setattr(PA, "_block_attention_ref", boom)
    monkeypatch.setattr(_ext(), "decode_attention_paged", boom)
    monkeypatch.setattr(_ext(), "attention_fwd_paged", boom)
    monkeypatch.setattr(_ext(), "decode_attention_paged_multi", boom)
    kernels.reset_launch_count()
    out, _, _, _ = PA.block_attention(qkv, kc, vc, *args, shared_prefix=sp)
    assert kernels.launch_count() == 2
    assert torch.isfinite(out.as_subclass(torch.Tensor).float()).all()


def test_shared_decode_kernels_use_no_local_memory():
    obj = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "paddle_b200", "_build_cache", "decode_attention.cuda.o")
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    shared = [f for f in funcs if "decode_shared" in f.split("\n", 1)[0]]
    assert len(shared) == 8                                       # split kernels (2 dtypes x 16-bit / int8 / fp8) and 2 merge kernels
    for f in shared:
        name = f.split("\n", 1)[0]
        assert "decode_multi" not in name
        assert not re.search(r"\b(LDL|STL)\b", f), name
        if "split_kernel" in name:
            assert re.search(r"\bHMMA\.16816\.F32", f), name
            assert "WARPGROUP" not in f, name


def test_engine_logits_with_prefix_caching_match_an_engine_without(monkeypatch):
    monkeypatch.setattr(PA, "SHARED_PREFIX_MIN_GROUP", 2)       # group every decode step of these few requests
    monkeypatch.setattr(PA, "SHARED_PREFIX_MIN_TOKENS", 16)
    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = models.llama_tiny(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                                vocab_size=512, max_position_embeddings=1024)
        m = models.LlamaForCausalLM(cfg)
    finally:
        paddle.set_default_dtype("float32")
        paddle.set_device("cpu")
    g = torch.Generator().manual_seed(0)
    system = torch.randint(1, cfg.vocab_size, (200,), generator=g).tolist()
    prompts = [system + torch.randint(1, cfg.vocab_size, (n,), generator=g).tolist() for n in (5, 9, 17, 2)]
    n = 8

    def serve(caching):
        eng = models.LLMEngine(m, num_blocks=128, block_size=16, enable_prefix_caching=caching)
        logits = {}
        fwd = eng._forward

        def record(seqs, n_new, enc, dec):
            out = fwd(seqs, n_new, enc, dec)
            for i, (s, k) in enumerate(zip(seqs, n_new)):
                logits[(s.id, s.cached + k)] = out[i].float()
            return out

        eng._forward = record
        ids = [eng.add_request(prompts[0], n)]
        eng.step()
        ids += [eng.add_request(p, n) for p in prompts[1:]]
        res = eng.run_until_done()
        return [res[i] for i in ids], logits, eng

    ref, ref_logits, _ = serve(False)
    out, logits, eng = serve(True)
    assert eng.stats["prefix_hit_tokens"] == 3 * 192
    checked = 0
    for i, p in enumerate(prompts):
        assert rel_err(logits[(i, len(p))], ref_logits[(i, len(p))]) < 2e-2, i        # the first token after a hit
        for j in range(1, n):                                    # decode steps (grouped) while both engines saw the same tokens
            if out[i][:j] != ref[i][:j]:
                break
            assert rel_err(logits[(i, len(p) + j)], ref_logits[(i, len(p) + j)]) < 2e-2, (i, j)
            checked += 1
    assert checked >= 8
