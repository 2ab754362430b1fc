"""int8 x int8 GEMM with exact int32 accumulation, and the per-token int8 activation quantizer (llm.int8 / W8A8 inference).

CUDA path: csrc/gemm_fp8_sm100.cu (gemm_s8_kernel: IGMMA, s32 accumulators, an int32 or a dequantising epilogue) and csrc/quant_fp8.cu
(quantize_rows_s8_kernel).  Both operands are K-major (a [M,K], b [N,K]: the [out, in] layout of `weight_quantize`).  CPU tensors run the
torch expressions below, which define the results: the kernels reproduce them bit for bit."""
from __future__ import annotations

import torch

from . import ext, raw, use_fused


def _aligned(t):
    """Contiguous with a 16-byte aligned base (the TMA / vector-load rule); copies only when needed."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def matmul_exact(x, y):
    """int32 x @ y of integer tensors through float64: exact while every |sum| < 2^53 (any int8 operands up to K = 2^38)."""
    return torch.matmul(x.double(), y.double()).to(torch.int32)


def gemm_int8(a, b):
    """a [M,K] / [B,M,K] int8, b [N,K] / [B,N,K] int8 -> a @ b^T, int32 and exact."""
    a, b = raw(a), raw(b)
    if use_fused(a) and a.shape[-1] % 16 == 0 and a.shape[-1] > 0:
        return ext().gemm_int8(_aligned(a), _aligned(b))
    return matmul_exact(a, b.transpose(-1, -2))


def gemm_int8_dequant(a, b, row_scale, col_scale, bias=None, out_dtype=torch.float32):
    """a [M,K], b [N,K] int8 -> (float(a @ b^T) * row_scale[m]) * col_scale[n] (+ bias[n]), each step rounded in fp32, then out_dtype."""
    a, b, row_scale, col_scale, bias = raw(a), raw(b), raw(row_scale), raw(col_scale), raw(bias)
    rs, cs = row_scale.float().reshape(-1).contiguous(), col_scale.float().reshape(-1).contiguous()
    bf = None if bias is None else bias.float().reshape(-1).contiguous()
    if use_fused(a) and a.shape[-1] % 16 == 0 and a.shape[-1] > 0:
        return ext().gemm_int8_dequant(_aligned(a), _aligned(b), rs, cs, bf, out_dtype)
    out = matmul_exact(a, b.t()).float() * rs.unsqueeze(1) * cs
    if bf is not None:
        out = out + bf
    return out.to(out_dtype)


def quantize_int8_rows(x, mask=None):
    """Per-token int8 of x [M, K] (bf16 / fp16 / fp32), in fp32: row_scale = max(absmax_row, 1e-8) / 127 and
    q = clamp(round_half_even(x / row_scale), -128, 127).  Columns where `mask` (bool [K]) is set are excluded from the scale and
    written as 0.  Returns (q int8 [M, K], row_scale fp32 [M]); on CUDA one launch and no host read."""
    x, mask = raw(x), raw(mask)
    if use_fused(x) and x.dim() == 2 and x.shape[1] % 16 == 0 and x.shape[1] > 0 and x.dtype in (torch.bfloat16, torch.float16, torch.float32):
        return tuple(ext().quantize_int8_rows(_aligned(x), None if mask is None else mask.to(torch.bool).contiguous()))
    xf = x.float()
    if mask is not None:
        xf = xf.masked_fill(mask.to(torch.bool), 0.0)
    sx = xf.abs().amax(-1, keepdim=True).clamp(min=1e-8) / 127.0
    q = torch.round(xf / sx).clamp(-128, 127).to(torch.int8)
    return q, sx.reshape(-1)
