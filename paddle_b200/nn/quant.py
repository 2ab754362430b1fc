"""Weight-only / llm.int8 quantised linear. Parity: python/paddle/nn/quant/quantized_linear.py
(weight_quantize, weight_dequantize, weight_only_linear, llm_int8_linear)."""
from __future__ import annotations

import torch

from ..tensor import Tensor


def _w(t):
    return t.as_subclass(Tensor) if isinstance(t, torch.Tensor) and not isinstance(t, Tensor) else t


def weight_quantize(x, algo="weight_only_int8", arch=None, group_size=-1):
    """x: [in, out] -> (int8 weight [out, in] (int4 packed two per byte), scale [out] or [groups, out])."""
    w = x.as_subclass(torch.Tensor).float()
    bits = 4 if "int4" in algo else 8
    qmax = 2 ** (bits - 1) - 1
    if group_size and group_size > 0:
        k, n = w.shape
        wg = w.reshape(k // group_size, group_size, n)
        scale = wg.abs().amax(1).clamp(min=1e-8) / qmax
        q = torch.round(wg / scale.unsqueeze(1)).clamp(-qmax - 1, qmax).reshape(k, n)
    else:
        scale = w.abs().amax(0).clamp(min=1e-8) / qmax
        q = torch.round(w / scale).clamp(-qmax - 1, qmax)
    q = q.t().contiguous().to(torch.int8)
    if bits == 4:
        lo, hi = q[:, 0::2] & 0xF, q[:, 1::2] & 0xF
        q = (lo | (hi << 4)).to(torch.int8)
    return _w(q), _w(scale.to(x.dtype if x.dtype != torch.float32 else torch.float32))


def _dequantize_torch(q, s, int4, dtype, group_size):
    """The reference expression: float(q) * float(scale), rounded once to `dtype`.  q [out, in] (int4 packed [out, in / 2]) -> [in, out],
    contiguous like the CUDA kernel's result and a Linear's weight, so both devices run the same GEMM on it."""
    if int4:
        lo = (q << 4).to(torch.int8) >> 4
        hi = q >> 4
        q = torch.stack([lo, hi], -1).reshape(q.shape[0], -1)
    w = q.float().t()
    s = s.float()
    if group_size and group_size > 0:
        w = (w.reshape(-1, group_size, w.shape[1]) * s.unsqueeze(1)).reshape(w.shape)
    else:
        w = w * s
    return w.to(dtype).contiguous()


def weight_dequantize(x, scale, algo="weight_only_int8", out_dtype="float16", group_size=-1):
    """x int8 [out, in] (int4: [out, in / 2]) and scale [out] or [in / group_size, out] -> [in, out] in out_dtype.  CUDA weights with a
    bf16 / fp16 / fp32 output run one kernel (csrc/gemm_wo_sm100.cu: reads the quantised weight once, writes the result once) that gives the
    same bits as the torch expression, which otherwise expands the weight through fp32 temporaries."""
    from ..framework.dtype import convert_dtype

    q = x.as_subclass(torch.Tensor)
    s = scale.as_subclass(torch.Tensor)
    dtype = convert_dtype(out_dtype)
    int4 = "int4" in algo
    if q.is_cuda and s.is_cuda and q.dtype == torch.int8 and q.dim() == 2 and dtype in (torch.bfloat16, torch.float16, torch.float32):
        from .._build import ext

        gs = int(group_size) if group_size and group_size > 0 else -1
        return _w(ext().weight_dequantize(q.contiguous(), s.float().contiguous(), int4, gs, dtype))
    return _w(_dequantize_torch(q, s, int4, dtype, group_size))


def weight_only_linear(x, weight, bias=None, weight_scale=None, weight_dtype="int8", arch=None, group_size=-1):
    """y = x @ dequant(weight)^T + bias.  CUDA bf16 / fp16 activations with per-channel or group-wise (group_size 64 / 128) scales run
    csrc/gemm_wo_sm100.cu: the int8 / int4 weights are streamed by TMA and expanded to 16-bit INSIDE the SM (no dequantised copy of the
    weight is ever written to HBM), which is what makes weight-only decoding faster than the 16-bit GEMM (it is bound by weight bytes).
    More than 64 rows: one dequantisation kernel + the 16-bit GEMM.  Other group sizes / CPU: dequantise + linear."""
    xr = x.as_subclass(torch.Tensor)
    wr = weight.as_subclass(torch.Tensor)
    per_channel = group_size is None or group_size <= 0
    if xr.is_cuda and xr.dtype in (torch.bfloat16, torch.float16) and weight_scale is not None and (per_channel or group_size in (64, 128)) \
            and weight_dtype in ("int8", "int4") and wr.dtype == torch.int8 and xr.shape[-1] % (64 if per_channel else max(64, group_size)) == 0 \
            and wr.shape[0] % 8 == 0:
        from ..framework.flags import flag

        if flag("FLAGS_use_fused_kernels", True):
            from .._build import ext

            x2 = xr.reshape(-1, xr.shape[-1]).contiguous()
            if x2.shape[0] > 64:
                # prefill: compute bound, and every token tile would dequantise the weight tile again - expand the weight once instead
                # (one pass over the int weights) and run the bf16 tcgen05 GEMM; the fused kernel is the decode / small-batch path
                w = weight_dequantize(weight, weight_scale, "weight_only_" + weight_dtype, x.dtype, group_size)
                from . import functional as F

                return F.linear(x, w, bias)
            sc = weight_scale.as_subclass(torch.Tensor).float().contiguous()
            b = None if bias is None else bias.as_subclass(torch.Tensor).to(xr.dtype).contiguous()
            y = ext().weight_only_gemm(x2, wr.contiguous(), sc, b, weight_dtype == "int4", -1 if per_channel else int(group_size))
            return _w(y.reshape(*xr.shape[:-1], wr.shape[0]))
    w = weight_dequantize(weight, weight_scale, "weight_only_" + weight_dtype, x.dtype, group_size)
    from . import functional as F

    return F.linear(x, w, bias)


def llm_int8_linear(x, weight, bias=None, weight_scale=None, threshold=6.0):
    """LLM.int8(): y = x @ dequant(weight)^T + bias with int8 activations.  weight int8 [out, in] and weight_scale fp32 [out] come from
    `weight_quantize(algo="llm.int8")`.  Outlier columns (any |x| > threshold over all rows) stay in x's dtype and are multiplied with
    their dequantised weight rows in fp32; the other columns are quantised per token (kernels.gemm_int8.quantize_int8_rows) and run
    through the int8 GEMM with exact integer sums, dequantised as (float(acc) * row_scale[m]) * weight_scale[n].  The two parts are
    added in fp32, then the bias, and the result is cast once to x's dtype.

    CUDA bf16 / fp16 activations (in % 16 == 0) run the sm_90a kernels.  A finite threshold reads the number of outlier columns on the
    host once per call; threshold=float("inf") skips outlier detection entirely: two launches (quantizer, int8 GEMM) and no host read,
    the path to use for serving."""
    from ..kernels import gemm_int8 as G8

    xr, wr = x.as_subclass(torch.Tensor), weight.as_subclass(torch.Tensor)
    ws = weight_scale.as_subclass(torch.Tensor).float()
    br = None if bias is None else bias.as_subclass(torch.Tensor)
    k = xr.shape[-1]
    x2 = xr.reshape(-1, k)
    no_outliers = threshold == float("inf")
    if xr.is_cuda and xr.dtype in (torch.bfloat16, torch.float16) and wr.dtype == torch.int8 and k % 16 == 0:
        from ..framework.flags import flag

        if flag("FLAGS_use_fused_kernels", True):
            if no_outliers:
                xq, sx = G8.quantize_int8_rows(x2)
                y = G8.gemm_int8_dequant(xq, wr, sx, ws, br, xr.dtype)
                return _w(y.reshape(*xr.shape[:-1], wr.shape[0]))
            outlier = (x2.abs() > threshold).any(0)
            xq, sx = G8.quantize_int8_rows(x2, outlier)
            out = G8.gemm_int8_dequant(xq, wr, sx, ws, None, torch.float32)
            idx = outlier.nonzero().flatten()                   # the one host read: the outlier count
            if idx.numel():
                from ..kernels.gemm import gemm

                pad = (-idx.numel()) % 8                        # zero columns / rows keep the 16-byte TMA granularity
                xo = torch.nn.functional.pad(x2[:, idx], (0, pad)).contiguous()
                wo = torch.nn.functional.pad(_dequantize_torch(wr[:, idx], ws, False, xr.dtype, -1), (0, 0, 0, pad)).contiguous()
                gemm(xo, wo, epilogue=4, out=out)                # out += x_outlier @ w_outlier, summed in fp32
            if br is not None:
                out = out + br.float()
            return _w(out.to(xr.dtype).reshape(*xr.shape[:-1], wr.shape[0]))
    outlier = torch.zeros(k, dtype=torch.bool, device=xr.device) if no_outliers else (x2.abs() > threshold).any(0)
    xq, sx = G8.quantize_int8_rows(x2, outlier)
    out = G8.matmul_exact(xq, wr.t()).float() * sx.unsqueeze(1) * ws
    w = weight_dequantize(weight, weight_scale, "weight_only_int8", x.dtype).as_subclass(torch.Tensor)
    out = out + x2[:, outlier].float() @ w[outlier].float()
    if br is not None:
        out = out + br.float()
    return _w(out.to(x.dtype).reshape(*xr.shape[:-1], wr.shape[0]))


def apply_per_channel_scale(x, scales):
    return x * scales


class Stub:
    """Placeholder marking where an observer / quanter is inserted by QAT / PTQ. Parity: nn/quant/stub.py:Stub."""

    def __init__(self, observer=None):
        self._observer = observer

    def __call__(self, x):
        return x

    forward = __call__


# static programs record these as single ops (their bodies compute on raw tensors; framework/recording.py)
from ..framework.recording import make_recordable as _make_recordable  # noqa: E402

_make_recordable(globals(), ['weight_quantize', 'weight_dequantize', 'llm_int8_linear', 'apply_per_channel_scale'])
