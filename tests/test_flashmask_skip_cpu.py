"""Tile skipping for column-masked attention, without a GPU:

- attention_flashmask_sm100.cuda.o, read with `cuobjdump -sass`, holds exactly the tile-skipping kernels (forward, dK/dV with and without
  the dQ stage, deterministic dQ; bf16 / fp16, head_dim 64 / 128, with and without dropout), the tile-summary kernel and the stats
  kernels; none touches local memory and every wgmma kernel keeps its MMAs pipelined;
- kernels.attention.colmask_tile_classes, the torch twin of the kernels' tile classes, against colmask_to_dense: a hidden tile has no
  visible element, an open tile no hidden one, and causal documents on 128-row boundaries cost exactly their own causal tiles;
- the column mask of flash_attn_unpadded for q and k packed differently under a causal mask;
- LlamaForCausalLM on packed documents (attn_mask_startend_row_indices, document-local position_ids) against each document run alone.
"""
import os
import shutil

import pytest
import torch

from paddle_b200.kernels import attention as KAT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "paddle_b200", "_build_cache", "attention_flashmask_sm100.cuda.o")
_sass = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(OBJ),
                           reason="cuobjdump, cu++filt or the built object is missing")

DTYPES = ("__nv_bfloat16", "__half")
B = ("(bool)0", "(bool)1")
INT_MAX = 2 ** 31 - 1


def _counts():
    from test_attention_d64_train_cpu import _counts as counts

    return counts(OBJ)


def _expected():
    out = {"b200::mask_skip::mask_tiles_kernel"}
    for t in DTYPES:
        for d in (64, 128):
            for p in B:
                out.add(f"void b200::attn::fwd_skip_kernel<{t}, (int){d}, {p}>")
                out.add(f"void b200::attn_bwd::dq_skip_kernel<{t}, (int){d}, {p}>")
                for dq in B:
                    out.add(f"void b200::attn_bwd::dkv_skip_kernel<{t}, {dq}, (int){d}, {p}>")
        for z in B:   # the stats kernels of the backward are the unmasked ones
            out.add(f"void b200::attn_bwd::prep_kernel<{t}, {z}>")
            out.add(f"void b200::attn_bwd::prep_d64_kernel<{t}, {z}>")
    return out


def _name(n):
    return n[:n.index(">(") + 1] if ">(" in n else n[:n.index("(")]


@_sass
def test_object_holds_exactly_the_skipping_kernels():
    names = {_name(n) for n in _counts()}
    assert names == _expected(), sorted(names ^ _expected())


@_sass
def test_skipping_kernels_use_no_local_memory():
    for n, c in _counts().items():
        assert c["local"] == 0, (n, c)


@_sass
def test_skipping_wgmma_kernels_are_pipelined():
    wgmma = {n: c for n, c in _counts().items() if "prep_" not in n and "mask_tiles" not in n}
    assert len(wgmma) == 32, sorted(wgmma)
    for n, c in wgmma.items():
        assert c["mma"] > 0 and c["arrive"] < c["mma"], (n, c)


# ---------------------------------------------------------------------------------------------------- tile classes
def _docs_colmask(b, lens, causal=True):
    """flashmask's causal document mask (key j hides the rows >= the end of its document) as the kernels' int4 form."""
    ends = torch.cat([torch.full((n,), e, dtype=torch.int32) for n, e in zip(lens, torch.tensor(lens).cumsum(0).tolist())])
    se = ends.reshape(1, 1, -1, 1).expand(b, 1, -1, 1).contiguous()
    return KAT.colmask_from_startend(se, causal, ends.numel())


def _random_colmask(g, b, hm, sq, sk):
    """Random 4-bound masks with both intervals, some keys hiding nothing, some everything."""
    lts = torch.randint(0, sq + 1, (b, hm, sk), generator=g)
    lte = (lts + torch.randint(0, sq + 1, (b, hm, sk), generator=g)).clamp(max=sq + 5)
    uts = torch.randint(0, sq + 1, (b, hm, sk), generator=g)
    ute = (uts + torch.randint(0, sq // 2 + 1, (b, hm, sk), generator=g)).clamp(max=sq)
    none = torch.rand(b, hm, sk, generator=g) < 0.1
    lts, uts = torch.where(none, sq + 9, lts), torch.where(none, 0, uts)
    ute = torch.where(none, 0, ute)
    return torch.stack([lts, lte, uts, ute], -1).int().contiguous()


def _block_structured(g, b, hm, sq, sk):
    """Masks whose bounds are constant over runs of keys, so that whole tiles come out hidden or open."""
    step = 96
    base = _random_colmask(g, b, hm, sq, -(-sk // step))
    return base.repeat_interleave(step, 2)[:, :, :sk].contiguous()


def _check_classes(cm, sq, sk, bm, bn, causal):
    cls = KAT.colmask_tile_classes(cm, sq, sk, bm, bn, causal)
    vis = KAT.colmask_to_dense(cm, sq)                                   # [b, hm, sq, sk]
    hid = ~vis
    if causal:
        cmask = torch.ones(sq, sk, dtype=torch.bool).tril(sk - sq)
        vis = vis & cmask
    nm, nn = cls.shape[2], cls.shape[3]
    pad = lambda t, v: torch.nn.functional.pad(t, (0, nn * bn - sk, 0, nm * bm - sq), value=v)  # noqa: E731
    tiles = lambda t: t.reshape(t.shape[0], t.shape[1], nm, bm, nn, bn).transpose(3, 4)       # noqa: E731
    any_vis = tiles(pad(vis, False)).any(-1).any(-1)
    any_hid = tiles(pad(hid[..., :sk], False)).any(-1).any(-1)
    assert not (any_vis & (cls == 0)).any(), "a hidden tile has a visible element"
    assert not (any_hid & (cls == 2)).any(), "an open tile has a hidden element"
    return cls


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("bm", [64, 128])
@pytest.mark.parametrize("kind", ["docs", "window", "random", "blocks"])
@pytest.mark.parametrize("sq,sk,hm", [(512, 512, 1), (700, 700, 3), (300, 555, 1), (1000, 389, 2)])
def test_tile_classes_against_dense(kind, bm, causal, sq, sk, hm):
    g = torch.Generator().manual_seed(sq * 7 + sk + hm)
    b = 2
    if kind == "docs":
        cuts = sorted(torch.randint(1, sk, (5,), generator=g).tolist())
        lens = [y - x for x, y in zip([0] + cuts, cuts + [sk]) if y > x]
        cm = _docs_colmask(b, lens, causal).expand(b, hm, sk, 4).contiguous()
    elif kind == "window":
        cm = KAT.colmask_from_window(sq, sk, 200, 0 if causal else 150, causal, "cpu").expand(b, hm, sk, 4).contiguous()
    elif kind == "random":
        cm = _random_colmask(g, b, hm, sq, sk)
    else:
        cm = _block_structured(g, b, hm, sq, sk)
    cls = _check_classes(cm, sq, sk, bm, 128, causal)
    if kind == "window" and causal and sk >= 512:
        assert (cls == 0).any(), "no tile was skipped"


def _doc_tiles(lens, bm=128, bn=128):
    """Tiles a causal call on each document alone computes (the dense kernels walk key tiles up to the causal limit)."""
    return sum(sum(min(-(-n // bn), (mt * bm + bm - 1) // bn + 1) for mt in range(-(-n // bm))) for n in lens)


@pytest.mark.parametrize("lens", [[1024] * 4, [256] * 16, [512, 1536, 128, 1920, 384, 640]])
@pytest.mark.parametrize("bm", [64, 128])
def test_aligned_documents_cost_their_own_tiles(lens, bm):
    s = sum(lens)
    cm = _docs_colmask(1, lens)
    cls = _check_classes(cm, s, s, bm, 128, True)
    assert int((cls != 0).sum()) == _doc_tiles(lens, bm)
    assert not (cls == 1).any(), "aligned documents leave no partial tile"


def test_expected_tile_counts():
    """The counts the forward computes per (batch, head), from shapes."""
    assert int((KAT.colmask_tile_classes(_docs_colmask(1, [1024] * 4), 4096, 4096, 128, 128, True) != 0).sum()) == 144
    assert int((KAT.colmask_tile_classes(_docs_colmask(1, [256] * 16), 4096, 4096, 128, 128, True) != 0).sum()) == 48
    win = KAT.colmask_from_window(16384, 16384, 4095, 0, True, "cpu")
    assert int((KAT.colmask_tile_classes(win, 16384, 16384, 128, 128, True) != 0).sum()) == 3696


# ---------------------------------------------------------------------------------------------------- varlen, different packings
def test_varlen_causal_mask_for_different_packings():
    cu_q = torch.tensor([0, 5, 5, 40, 41, 90], dtype=torch.int32)
    cu_k = torch.tensor([0, 9, 12, 40, 70, 101], dtype=torch.int32)
    tq, tk = int(cu_q[-1]), int(cu_k[-1])
    ref = torch.zeros(tq, tk, dtype=torch.bool)
    for s in range(len(cu_q) - 1):
        q0, q1, k0, k1 = (int(x) for x in (cu_q[s], cu_q[s + 1], cu_k[s], cu_k[s + 1]))
        lq, lk = q1 - q0, k1 - k0
        for i in range(lq):
            for j in range(lk):
                ref[q0 + i, k0 + j] = j <= i + lk - lq
    cm = KAT.colmask_from_cu_seqlens(cu_q, cu_k, tk + 3, causal=True)      # 3 keys past the last sequence hide every row
    vis = KAT.colmask_to_dense(cm, tq)[0, 0]
    assert torch.equal(vis[:, :tk], ref)
    assert not vis[:, tk:].any()


# ---------------------------------------------------------------------------------------------------- Llama on packed documents
def _llama(recompute, window=None, seed=0):
    import paddle_b200 as paddle
    from paddle_b200.models import LlamaForCausalLM, llama_tiny

    paddle.seed(seed)
    cfg = llama_tiny(num_attention_heads=4, num_key_value_heads=2, recompute=recompute, sliding_window=window, dtype="float32")
    return LlamaForCausalLM(cfg), cfg


def _grads(model):
    return {n: p.grad.as_subclass(torch.Tensor).clone() for n, p in model.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("recompute,window", [(False, None), (True, None), (False, 5), (True, 7)])
def test_llama_documents_match_separate_runs(recompute, window):
    import paddle_b200 as paddle

    paddle.set_default_dtype("float32")
    model, cfg = _llama(recompute, window)
    model.train()
    g = torch.Generator().manual_seed(1)
    lens = [[7, 13, 12], [32]]
    s = 32
    ids = torch.randint(0, cfg.vocab_size, (2, s + 1), generator=g)
    x, y = ids[:, :-1], ids[:, 1:].clone()
    ends = torch.stack([torch.cat([torch.full((n,), e) for n, e in zip(row, torch.tensor(row).cumsum(0).tolist())]) for row in lens])
    pos = torch.stack([torch.cat([torch.arange(n) for n in row]) for row in lens])
    for r, row in enumerate(lens):   # a document's last label would be the next document's first token: not a target
        for e in torch.tensor(row).cumsum(0).tolist()[:-1]:
            y[r, e - 1] = -100
    se = ends.reshape(2, 1, s, 1).int()
    P = lambda t: t.as_subclass(paddle.Tensor)  # noqa: E731
    logits = model(P(x), None, P(pos), P(se)).as_subclass(torch.Tensor)
    loss = model(P(x), P(y), P(pos), P(se))
    loss.backward()
    packed = _grads(model)
    model.clear_gradients()

    total, n_tok, ref_logits = 0.0, 0, []
    for r, row in enumerate(lens):
        st = 0
        for n in row:
            xi, yi = x[r:r + 1, st:st + n], y[r:r + 1, st:st + n]
            ref_logits.append(model(P(xi)).as_subclass(torch.Tensor)[0])
            valid = int((yi != -100).sum())
            li = model(P(xi), P(yi))
            (li * valid).backward()
            total += float(li) * valid
            n_tok += valid
            st += n
    sep = {k: v / n_tok for k, v in _grads(model).items()}
    torch.testing.assert_close(logits.reshape(-1, logits.shape[-1]), torch.cat(ref_logits).reshape(-1, logits.shape[-1]), rtol=1e-4, atol=1e-5)
    assert abs(float(loss) - total / n_tok) < 1e-5
    assert packed.keys() == sep.keys()
    for k in packed:
        torch.testing.assert_close(packed[k], sep[k], rtol=1e-4, atol=1e-6, msg=k)


def test_llama_without_documents_keeps_its_path(monkeypatch):
    """No attn_mask_startend_row_indices: the layers are called as before, without a column mask."""
    import paddle_b200 as paddle
    from paddle_b200.models import llama as L

    paddle.set_default_dtype("float32")
    model, cfg = _llama(False)
    seen = []
    orig = L.LlamaAttention.attend

    def attend(self, qkv, cos, sin, position_ids=None, colmask=None):
        seen.append(colmask)
        return orig(self, qkv, cos, sin, position_ids, colmask)

    monkeypatch.setattr(L.LlamaAttention, "attend", attend)
    model(paddle.randint(0, cfg.vocab_size, [1, 16]))
    assert seen and all(c is None for c in seen)
