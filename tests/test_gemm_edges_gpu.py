"""The persistent GEMM at its tile edges, against an fp32 torch reference: odd and single M-tile counts, ragged M / N / K, more work
than resident CTAs (each loops over tiles), every epilogue, accumulation into an existing bf16 D (old D loaded two boxes ahead of the
epilogue), strided batches and both grouped (MoE) modes with skipped experts."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ext():
    from paddle_b200._build import ext

    return ext()


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _gemm(A, B, a_km, b_nk, **kw):
    a_in = A.t().contiguous() if a_km else A
    b_in = B.t().contiguous() if b_nk else B
    assert _ext().gemm_supported(a_in, b_in, a_km, b_nk)
    return _ext().gemm(a_in, b_in, kw.get("bias"), a_km, b_nk, kw.get("epilogue", 0), kw.get("out"), kw.get("out_dtype"))


@pytest.mark.parametrize("a_km,b_nk", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("m,n,k", [
    (384, 512, 256),      # odd number of M-tiles
    (128, 768, 320),      # one M-tile
    (648, 1000, 200),     # M, N and K all ragged (N not a multiple of the tile width, K not of 64)
    (96, 256, 128),       # less than one M-tile
    (4224, 4352, 192),    # 33 x 17 tiles: more tiles than SMs, odd M-tile count
])
def test_gemm_edge_layouts(a_km, b_nk, m, n, k):
    torch.manual_seed(0)
    A = torch.randn(m, k, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(k, n, device="cuda", dtype=torch.bfloat16)
    out = _gemm(A, B, a_km, b_nk)
    assert out.shape == (m, n)
    assert rel_err(out, A.float() @ B.float()) < 5e-3


@pytest.mark.parametrize("m", [384, 128, 520])
def test_gemm_edge_epilogues(m):
    torch.manual_seed(1)
    n, k = 776, 136
    A = torch.randn(m, k, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(k, n, device="cuda", dtype=torch.bfloat16)
    bias = torch.randn(n, device="cuda", dtype=torch.bfloat16)
    ref = A.float() @ B.float()
    assert rel_err(_gemm(A, B, False, False, bias=bias, epilogue=1), ref + bias.float()) < 5e-3
    assert rel_err(_gemm(A, B, False, False, bias=bias, epilogue=2), torch.nn.functional.gelu(ref + bias.float())) < 5e-3
    assert rel_err(_gemm(A, B, False, True, bias=bias, epilogue=3), torch.relu(ref + bias.float())) < 5e-3
    o32 = _gemm(A, B, False, False, out_dtype=torch.float32)
    assert o32.dtype == torch.float32 and rel_err(o32, ref) < 1e-3
    acc32 = torch.ones(m, n, device="cuda", dtype=torch.float32)
    _gemm(A, B, False, False, epilogue=4, out=acc32)
    assert rel_err(acc32, ref + 1) < 1e-3


@pytest.mark.parametrize("m,n,k", [(384, 512, 320), (1152, 4096, 256), (128, 256, 64)])
def test_gemm_edge_accumulate_bf16(m, n, k):
    """dW-style accumulate (A read as [K, M], B as [K, N]) into an existing bf16 D: fp32(acc) + fp32(old), rounded once."""
    torch.manual_seed(2)
    X = torch.randn(k, m, device="cuda", dtype=torch.bfloat16)
    dY = torch.randn(k, n, device="cuda", dtype=torch.bfloat16)
    G = (torch.randn(m, n, device="cuda") * 4).to(torch.bfloat16)
    want = (X.float().t() @ dY.float() + G.float())
    _ext().gemm(X, dY, None, True, False, 4, G, None)
    assert rel_err(G, want) < 5e-3


def test_gemm_edge_strided_batch():
    torch.manual_seed(3)
    b, m, n, k = 5, 384, 320, 192
    A = torch.randn(b, m, k + 64, device="cuda", dtype=torch.bfloat16)[:, :, :k]      # padded rows: lda = k + 64
    B = torch.randn(2 * b, n, k, device="cuda", dtype=torch.bfloat16)[::2]            # every other matrix: batch stride 2 n k
    out = _ext().gemm(A, B, None, False, True, 0, None, None)
    ref = torch.einsum("bmk,bnk->bmn", A.float(), B.float())
    assert rel_err(out, ref) < 5e-3


@pytest.mark.parametrize("b_nk", [False, True])
def test_gemm_edge_grouped_rows(b_nk):
    """Rows grouped by expert in 256-row blocks (an odd number of them), one block of padding skipped (-1)."""
    torch.manual_seed(4)
    E, k, n = 3, 192, 384
    te = torch.tensor([0, 2, 2, -1, 1], dtype=torch.int32, device="cuda")
    m = 256 * te.numel()
    A = torch.randn(m, k, device="cuda", dtype=torch.bfloat16)
    W = torch.randn(E, k, n, device="cuda", dtype=torch.bfloat16)
    w_in = W.transpose(1, 2).contiguous() if b_nk else W
    out = torch.full((m, n), 7.0, device="cuda", dtype=torch.bfloat16)
    _ext().gemm_grouped(A, w_in, te, b_nk, out)
    for blk, e in enumerate(te.tolist()):
        rows = slice(256 * blk, 256 * blk + 256)
        if e < 0:
            assert bool((out[rows] == 7.0).all())       # a skipped block is left untouched
        else:
            assert rel_err(out[rows], A[rows].float() @ W[e].float()) < 5e-3


def test_gemm_edge_grouped_wgrad():
    """Per-expert weight gradients accumulated into [E, K_in, N]: an expert with no rows gets nothing added; K_in = 384 is an odd
    number of M-tiles."""
    torch.manual_seed(5)
    k_in, n = 384, 320
    rows = [192, 0, 64, 320]                  # expert 1 received no rows
    k0 = [0, 192, 192, 256]
    R = sum(rows)
    x = torch.randn(R, k_in, device="cuda", dtype=torch.bfloat16)
    dy = torch.randn(R, n, device="cuda", dtype=torch.bfloat16)
    out = torch.randn(len(rows), k_in, n, device="cuda").to(torch.bfloat16)
    before = out.float().clone()
    _ext().gemm_grouped_wgrad(x, dy, torch.tensor(k0, dtype=torch.int32, device="cuda"),
                              torch.tensor([r // 64 for r in rows], dtype=torch.int32, device="cuda"), out)
    for e, (r0, nr) in enumerate(zip(k0, rows)):
        want = before[e] + x[r0:r0 + nr].float().t() @ dy[r0:r0 + nr].float()
        if nr == 0:
            assert torch.equal(out[e].float(), before[e])
        else:
            assert rel_err(out[e], want) < 5e-3
