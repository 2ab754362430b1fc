"""Linear algebra. Parity: python/paddle/tensor/linalg.py."""
from __future__ import annotations

import torch

from ._helpers import T, ax, dt, raw, to_int, wrap


def matmul(x, y, transpose_x=False, transpose_y=False, name=None):
    """paddle.matmul. Parity: python/paddle/tensor/linalg.py:matmul -> phi MatmulKernel."""
    x, y = T(x), T(y)
    if transpose_x and x.dim() >= 2:
        x = torch.transpose(x, -1, -2)
    if x.dtype == torch.int8 and y.dtype == torch.int8:
        return _matmul_int8(x, y, transpose_y)
    if transpose_y and y.dim() >= 2:
        y = torch.transpose(y, -1, -2)
    from ..amp.auto_cast import _state, fp32_guard

    if _state["enabled"]:
        ctx, (x, y) = fp32_guard("matmul", x, y)
        with ctx:
            return torch.matmul(x, y)
    return torch.matmul(x, y)


def _matmul_int8(x, y, transpose_y):
    """int8 @ int8 -> int32, exact, on every device (the reference's cuBLASLt int8 -> int32 matmul).  CUDA 2-D operands and 3-D ones with
    one batch size run the int8 wgmma GEMM (kernels/gemm_int8.py), which takes B as [N, K]: transpose_y=True feeds y directly, otherwise
    one int8 copy of y^T is made.  Other shapes (K % 16 != 0, broadcasting, vectors) and CPU tensors: float64 product, exact while
    |sum| < 2^53."""
    from ..kernels import gemm_int8 as G8
    from ..kernels import use_fused

    if use_fused(x) and y.is_cuda and x.dim() == y.dim() and x.dim() in (2, 3) and (x.dim() == 2 or x.shape[0] == y.shape[0]) \
            and x.shape[-1] % 16 == 0 and x.shape[-1] > 0 and x.shape[-1] == y.shape[-1 if transpose_y else -2]:
        b = y if transpose_y else torch.transpose(y, -1, -2)
        return wrap(G8.gemm_int8(x.contiguous(), b.contiguous()))
    if transpose_y and y.dim() >= 2:
        y = torch.transpose(y, -1, -2)
    return wrap(G8.matmul_exact(x, y))


def mm(input, mat2, name=None):
    return torch.matmul(T(input), T(mat2))


def bmm(x, y, name=None):
    return torch.bmm(T(x), T(y))


def dot(x, y, name=None):
    x, y = T(x), T(y)
    return (x * y).sum(-1)


def mv(x, vec, name=None):
    return torch.mv(T(x), T(vec))


def vecdot(x, y, axis=-1, name=None):
    return torch.linalg.vecdot(T(x), T(y), dim=axis)


def cross(x, y, axis=9, name=None):
    x, y = T(x), T(y)
    if axis == 9:
        axis = next(i for i, s in enumerate(x.size()) if s == 3)
    return torch.cross(x, y, dim=axis)


def norm(x, p=None, axis=None, keepdim=False, name=None):
    x = T(x)
    a = ax(axis)
    if p is None:
        p = "fro" if (a is None or isinstance(a, tuple)) else 2
    if p == "fro":
        if a is None:
            return torch.sqrt(torch.sum(x * x)).reshape([1] * x.dim()) if keepdim else torch.sqrt(torch.sum(x.abs() ** 2))
        return torch.sqrt(torch.sum(x.abs() ** 2, dim=a, keepdim=keepdim))
    if p == "nuc":
        return torch.linalg.matrix_norm(x, "nuc", dim=a if a is not None else (-2, -1), keepdim=keepdim)
    if isinstance(a, tuple) and len(a) == 2 and p in (1, -1, 2, -2, float("inf"), float("-inf")):
        return torch.linalg.matrix_norm(x, p, dim=a, keepdim=keepdim)
    if a is None:
        out = torch.linalg.vector_norm(x.reshape(-1), p)
        return out.reshape([1] * x.dim()) if keepdim else out
    return torch.linalg.vector_norm(x, p, dim=a, keepdim=keepdim)


def vector_norm(x, p=2.0, axis=None, keepdim=False, name=None):
    return torch.linalg.vector_norm(T(x), p, dim=ax(axis), keepdim=keepdim)


def matrix_norm(x, p="fro", axis=(-2, -1), keepdim=False, name=None):
    return torch.linalg.matrix_norm(T(x), p, dim=tuple(axis), keepdim=keepdim)


def dist(x, y, p=2, name=None):
    return torch.dist(T(x), T(y), p)


def cdist(x, y, p=2.0, compute_mode="use_mm_for_euclid_dist_if_necessary", name=None):
    return torch.cdist(T(x), T(y), p)


def cholesky(x, upper=False, name=None):
    return torch.linalg.cholesky(T(x), upper=upper)


def cholesky_solve(x, y, upper=False, name=None):
    return torch.cholesky_solve(T(x), T(y), upper=upper)


def cholesky_inverse(x, upper=False, name=None):
    return torch.cholesky_inverse(T(x), upper=upper)


def qr(x, mode="reduced", name=None):
    q, r = torch.linalg.qr(T(x), mode=mode)
    return r if mode == "r" else (q, r)


def svd(x, full_matrices=False, name=None):
    u, s, vh = torch.linalg.svd(T(x), full_matrices=full_matrices)
    return u, s, vh


def svdvals(x, name=None):
    return torch.linalg.svdvals(T(x))


def svd_lowrank(x, q=None, niter=2, M=None, name=None):
    u, s, v = torch.svd_lowrank(raw(x), q=q if q is not None else min(6, *raw(x).shape[-2:]), niter=niter, M=None if M is None else raw(M))
    return wrap(u), wrap(s), wrap(v)


def pca_lowrank(x, q=None, center=True, niter=2, name=None):
    u, s, v = torch.pca_lowrank(raw(x), q=q, center=center, niter=niter)
    return wrap(u), wrap(s), wrap(v)


def eig(x, name=None):
    w, v = torch.linalg.eig(T(x))
    return w, v


def eigvals(x, name=None):
    return torch.linalg.eigvals(T(x))


def eigh(x, UPLO="L", name=None):
    w, v = torch.linalg.eigh(T(x), UPLO=UPLO)
    return w, v


def eigvalsh(x, UPLO="L", name=None):
    return torch.linalg.eigvalsh(T(x), UPLO=UPLO)


def inv(x, name=None):
    return torch.linalg.inv(T(x))


inverse = inv


def pinv(x, rcond=1e-15, hermitian=False, name=None):
    return torch.linalg.pinv(T(x), rcond=rcond, hermitian=hermitian)


def solve(x, y, left=True, name=None):
    return torch.linalg.solve(T(x), T(y), left=left)


def triangular_solve(x, y, upper=True, transpose=False, unitriangular=False, name=None):
    x = T(x)
    if transpose:
        x, upper = torch.transpose(x, -1, -2), not upper
    return torch.linalg.solve_triangular(x, T(y), upper=upper, unitriangular=unitriangular)


def lstsq(x, y, rcond=None, driver=None, name=None):
    xr, yr = raw(x), raw(y)
    r = torch.linalg.lstsq(xr, yr, rcond=rcond, driver=driver)
    sol = r.solution
    res = r.residuals
    if res.numel() == 0 and xr.shape[-2] > xr.shape[-1]:
        res = ((xr @ sol - yr) ** 2).sum(-2)
    rank = r.rank if r.rank.numel() else torch.linalg.matrix_rank(xr)
    sv = r.singular_values if r.singular_values.numel() else torch.linalg.svdvals(xr)
    return wrap(sol), wrap(res), wrap(rank), wrap(sv)


def lu(x, pivot=True, get_infos=False, name=None):
    LU, piv, info = torch.linalg.lu_factor_ex(T(x), pivot=pivot)
    return (LU, piv, info) if get_infos else (LU, piv)


def lu_unpack(x, y, unpack_ludata=True, unpack_pivots=True, name=None):
    p, l, u = torch.lu_unpack(T(x), T(y), unpack_data=unpack_ludata, unpack_pivots=unpack_pivots)
    return p, l, u


def lu_solve(b, lu, pivots, trans="N", name=None):
    return torch.linalg.lu_solve(T(lu), T(pivots), T(b), adjoint=(trans != "N"))


def det(x, name=None):
    return torch.linalg.det(T(x))


def slogdet(x, name=None):
    s, l = torch.linalg.slogdet(T(x))
    return torch.stack([s, l], 0)


def matrix_power(x, n, name=None):
    return torch.linalg.matrix_power(T(x), n)


def matrix_rank(x, tol=None, hermitian=False, atol=None, rtol=None, name=None):
    if tol is not None:
        return torch.linalg.matrix_rank(T(x), tol=to_int(tol), hermitian=hermitian)
    return torch.linalg.matrix_rank(T(x), atol=atol, rtol=rtol, hermitian=hermitian)


def matrix_exp(x, name=None):
    return torch.linalg.matrix_exp(T(x))


def multi_dot(x, name=None):
    return torch.linalg.multi_dot([T(i) for i in x])


def cond(x, p=None, name=None):
    return torch.linalg.cond(T(x), p)


def cov(x, rowvar=True, ddof=True, fweights=None, aweights=None, name=None):
    x = T(x)
    if not rowvar and x.dim() == 2:
        x = x.t()
    return torch.cov(x, correction=1 if ddof else 0, fweights=None if fweights is None else T(fweights), aweights=None if aweights is None else T(aweights))


def corrcoef(x, rowvar=True, name=None):
    x = T(x)
    if not rowvar and x.dim() == 2:
        x = x.t()
    return torch.corrcoef(x)


def householder_product(x, tau, name=None):
    return torch.linalg.householder_product(T(x), T(tau))


def ormqr(x, tau, y, left=True, transpose=False, name=None):
    return torch.ormqr(T(x), T(tau), T(y), left=left, transpose=transpose)


def bincount(x, weights=None, minlength=0, name=None):
    return torch.bincount(T(x), None if weights is None else T(weights), minlength)


def histogramdd(*a, **k):
    from .math import histogramdd as _h

    return _h(*a, **k)


def fp8_fp8_half_gemm_fused(x, y, transpose_x=False, transpose_y=False, bias=None, scale=1.0, output_dtype="float16", act="identity", name=None):
    """fp8 x fp8 -> half GEMM. Parity: python/paddle/tensor/linalg.py (paddle/phi/kernels/fusion/fp8_gemm)."""
    from ..kernels import gemm_fp8

    return gemm_fp8.fp8_gemm(x, y, transpose_x, transpose_y, bias, scale, dt(output_dtype), act)


__all__ = [n for n in list(globals()) if not n.startswith("_") and n not in ("torch", "T", "ax", "dt", "raw", "to_int", "wrap", "annotations")]


# static programs record these as single ops (their bodies compute on raw tensors / read values; framework/recording.py)
from ..framework.recording import make_recordable as _make_recordable  # noqa: E402

_make_recordable(globals(), ['histogramdd', 'lstsq', 'pca_lowrank', 'svd_lowrank'])
