"""Attention dropout without a GPU: the kernels read from the built object with `cuobjdump -sass` (attention_dropout_sm100.cuda.o holds
exactly the dropout forward, dK/dV with and without the dQ stage, dQ and stats kernels, none touches local memory and every wgmma kernel
keeps its MMAs pipelined), and the torch twin of the mask, kernels.attention.dropout_keep_mask: known answers against Philox4x32-10,
its keep rate, and the independence of masks drawn at other offsets and for other (batch, head) planes."""
import math
import os
import shutil

import pytest
import torch

from paddle_b200.kernels.attention import dropout_keep, dropout_keep_mask
from paddle_b200.kernels.sampling import philox4x32_10

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "paddle_b200", "_build_cache", "attention_dropout_sm100.cuda.o")
_sass = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(OBJ),
                           reason="cuobjdump, cu++filt or the built object is missing")

DTYPES = ("__nv_bfloat16", "__half")
B = ("(bool)0", "(bool)1")


def _counts():
    from test_attention_d64_train_cpu import _counts as counts

    return counts(OBJ)


def _expected():
    out = set()
    for t in DTYPES:
        for d in (64, 128):
            for m in B:
                out.add(f"void b200::attn::fwd_dropout_kernel<{t}, {m}, (int){d}>")
                out.add(f"void b200::attn_bwd::dq_dropout_kernel<{t}, {m}, (int){d}>")
                for dq in B:
                    out.add(f"void b200::attn_bwd::dkv_dropout_kernel<{t}, {m}, {dq}, (int){d}>")
            for z in B:   # the dropout-free stats kernels (delta on the dropped O is unchanged)
                out.add(f"void b200::attn_bwd::prep_kernel<{t}, {z}>")
                out.add(f"void b200::attn_bwd::prep_d64_kernel<{t}, {z}>")
    return out


@_sass
def test_dropout_object_holds_exactly_the_dropout_kernels():
    names = {n[:n.index(">(") + 1] for n in _counts()}
    assert names == _expected(), sorted(names ^ _expected())


@_sass
def test_dropout_kernels_use_no_local_memory():
    for n, c in _counts().items():
        assert c["local"] == 0, (n, c)


@_sass
def test_dropout_wgmma_kernels_are_pipelined():
    wgmma = {n: c for n, c in _counts().items() if "prep_" not in n}
    assert len(wgmma) == 32, sorted(wgmma)
    for n, c in wgmma.items():
        assert c["mma"] > 0 and c["arrive"] < c["mma"], (n, c)


def _draw(seed, offset, b, h, H, i, j):
    """One element's 16-bit draw, written out from the layout in csrc/include/b200_philox.cuh."""
    plane = offset + b * H + h
    rc = 8 * (i >> 4) + (i & 7)
    kc = 4 * (j >> 4) + ((j & 7) >> 1)
    w = philox4x32_10(seed & 0xFFFFFFFF, seed >> 32, kc, rc, plane & 0xFFFFFFFF, plane >> 32)
    word = int(w[2 * ((i >> 3) & 1) + ((j >> 3) & 1)])
    return (word >> (16 * (j & 1))) & 0xFFFF


@pytest.mark.parametrize("seed,offset", [(0, 0), (42, 7), (0x123456789ABC, 2 ** 33 + 5)])
def test_mask_known_answers(seed, offset):
    b, h, sq, sk, p = 2, 3, 40, 37, 0.1
    m = dropout_keep_mask(seed, offset, b, h, sq, sk, p)
    g = torch.Generator().manual_seed(seed % 1000)
    for _ in range(24):
        bi, hi, i, j = (int(torch.randint(0, n, (1,), generator=g)) for n in (b, h, sq, sk))
        assert bool(m[bi, hi, i, j]) == (_draw(seed, offset, bi, hi, h, i, j) < dropout_keep(p)), (bi, hi, i, j)


def test_no_two_elements_share_a_draw():
    """Every (query, key) of a 32 x 32 plane reads its own half-word: the (call, word, half) triples are distinct."""
    seen = set()
    for i in range(32):
        for j in range(32):
            t = (8 * (i >> 4) + (i & 7), 4 * (j >> 4) + ((j & 7) >> 1), 2 * ((i >> 3) & 1) + ((j >> 3) & 1), j & 1)
            assert t not in seen
            seen.add(t)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_rate(p):
    m = dropout_keep_mask(2024, 11, 4, 8, 560, 560, p)     # 1.0e7 elements
    n = m.numel()
    assert n >= 10 ** 7
    assert abs(dropout_keep(p) / 65536 - (1 - p)) <= 2 ** -17
    rate = m.double().mean().item()
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(rate - (1 - p)) < 5 * sigma, (rate, 1 - p, sigma)


def _agreement_ok(a, b, p):
    """a and b independent: they agree at the rate (1-p)^2 + p^2, within 5 sigma."""
    n = a.numel()
    e = (1 - p) ** 2 + p ** 2
    r = (a == b).double().mean().item()
    return abs(r - e) < 5 * math.sqrt(e * (1 - e) / n), (r, e)


def test_masks_at_other_offsets_and_planes_are_independent():
    p = 0.5
    base = dropout_keep_mask(7, 1000, 2, 2, 256, 256, p)
    later = dropout_keep_mask(7, 1000 + 4, 2, 2, 256, 256, p)        # the next call's offsets (B H = 4)
    ok, info = _agreement_ok(base, later, p)
    assert ok, info
    ok, info = _agreement_ok(base[0, 0], base[1, 1], p)               # distinct (batch, head) planes of one call
    assert ok, info
    ok, info = _agreement_ok(base[0, 0], base[0, 1], p)
    assert ok, info
    ok, info = _agreement_ok(base, dropout_keep_mask(8, 1000, 2, 2, 256, 256, p), p)
    assert ok, info
    # a plane is the same function of (seed, offset + b H + h) wherever it sits
    assert torch.equal(base[1, 0], dropout_keep_mask(7, 1002, 1, 1, 256, 256, p)[0, 0])
