"""fp8 GEMM (per-tensor scaled e4m3 / e5m2 -> half, and OCP MX block-scaled e4m3) and fp8 Linears for O2-fp8 training.
Parity: paddle.linalg.fp8_fp8_half_gemm_fused (python/paddle/tensor/linalg.py) -> phi fp8_gemm fusion kernels (cuBLASLt).

CUDA path: csrc/gemm_fp8_sm100.cu — fp8 wgmma MMAs, fp32 accumulation in registers, dequantisation scale + bias +
activation fused in the epilogue.  Both operands must be K-major (x [M,K], y [N,K], i.e. transpose_x=False, transpose_y=True);
other layouts are brought into that form with one transposed copy.  CPU / unsupported shapes: fp32 reference."""
from __future__ import annotations

import torch

from ..framework.recording import recordable
from . import ext, raw, use_fused, wrap

E4M3_MAX, E5M2_MAX = 448.0, 57344.0
_FP8 = (torch.float8_e4m3fn, torch.float8_e5m2)


def _ref(x, y, transpose_x, transpose_y, bias, scale, out_dtype, act):
    xf, yf = x.to(torch.float32), y.to(torch.float32)
    if transpose_x:
        xf = xf.transpose(-1, -2)
    if transpose_y:
        yf = yf.transpose(-1, -2)
    out = torch.matmul(xf, yf) * scale
    if bias is not None:
        out = out + bias.float()
    if act == "gelu":
        out = torch.nn.functional.gelu(out)
    elif act == "relu":
        out = torch.relu(out)
    return out.to(out_dtype or torch.float16)


@recordable
def fp8_gemm(x, y, transpose_x=False, transpose_y=False, bias=None, scale=1.0, out_dtype=torch.float16, act="identity"):
    x, y, bias = raw(x), raw(y), raw(bias)
    out_dtype = out_dtype or torch.float16
    if use_fused(x) and x.dtype in _FP8 and y.dtype in _FP8 and x.dim() == 2 and y.dim() == 2 and out_dtype in (torch.float16, torch.bfloat16, torch.float32):
        a = x.t().contiguous() if transpose_x else x.contiguous()            # [M, K]
        b = y.contiguous() if transpose_y else y.t().contiguous()            # [N, K]
        if a.shape[1] % 16 == 0 and a.shape[1] == b.shape[1] and b.shape[0] % 8 == 0:
            bb = bias.to(out_dtype).contiguous() if bias is not None else None
            return wrap(ext().gemm_fp8(a, b, bb, float(scale), {"identity": 0, None: 0, "gelu": 1, "relu": 2}[act], out_dtype))
    return wrap(_ref(x, y, transpose_x, transpose_y, bias, scale, out_dtype, act))


def quantize_fp8(t, dtype=torch.float8_e4m3fn, amax=None):
    """Per-tensor scaling: returns (t_fp8, inv_scale) with t ~= t_fp8 * inv_scale (inv_scale stays a device tensor on CUDA)."""
    t = raw(t)
    if amax is None and _fused_quant_ok(t):
        q, _, inv = ext().quantize_fp8(t.contiguous(), dtype == torch.float8_e5m2, False)
        return q, inv
    fmax = E4M3_MAX if dtype == torch.float8_e4m3fn else E5M2_MAX
    amax = t.detach().abs().amax().float().clamp_min(1e-12) if amax is None else amax
    scale = fmax / amax
    q = (t.float() * scale).clamp(-fmax, fmax).to(dtype)
    return q, (1.0 / scale)


def _fused_quant_ok(t):
    return use_fused(t) and t.dim() == 2 and t.dtype in (torch.bfloat16, torch.float16, torch.float32) and t.shape[0] % 64 == 0 and t.shape[1] % 64 == 0


def quantize_fp8_pair(t, dtype=torch.float8_e4m3fn):
    """(q [M,K], qT [K,M], inv_scale): the tensor and its transpose quantised in one pass (csrc/quant_fp8.cu), scale on the device."""
    t = raw(t)
    if _fused_quant_ok(t):
        q, qt, inv = ext().quantize_fp8(t.contiguous(), dtype == torch.float8_e5m2, True)
        return q, qt, inv
    q, inv = quantize_fp8(t, dtype)
    return q, q.t().contiguous(), inv


def _scaled_gemm(a, b, sa, sb, bias, out_dtype):
    """a [M,K] fp8, b [N,K] fp8, sa / sb dequantisation factors (device tensors or floats) -> [M,N]."""
    if use_fused(a) and isinstance(sa, torch.Tensor) and isinstance(sb, torch.Tensor) and a.shape[1] % 16 == 0 and b.shape[0] % 8 == 0:
        bb = bias.to(out_dtype).contiguous() if bias is not None else None
        return ext().gemm_fp8(a, b, bb, 1.0, 0, out_dtype, sa.reshape(1).float(), sb.reshape(1).float())
    scale = (sa if isinstance(sa, torch.Tensor) else torch.tensor(float(sa))) * (sb if isinstance(sb, torch.Tensor) else torch.tensor(float(sb)))
    out = torch.matmul(a.float(), b.float().t()) * scale.to(a.device).float()
    if bias is not None:
        out = out + bias.float()
    return out.to(out_dtype)


class _Fp8Linear(torch.autograd.Function):
    """y = x @ W (W: [in, out]) with e4m3 activations / weights in the forward and e5m2 output gradients in the backward (the fp8 recipe of
    the reference's O2-fp8 AMP): three wgmma fp8 GEMMs, all TN.  Every operand is quantised ONCE by the fused kernels, which emit the
    transposed copy in the same pass; the dequantisation factors never leave the device."""

    @staticmethod
    def forward(ctx, x, w, bias):
        x2 = x.reshape(-1, x.shape[-1])
        xq, xqt, sx = quantize_fp8_pair(x2)              # [M, in], [in, M]
        wq, wqt, sw = quantize_fp8_pair(w)               # [in, out], [out, in]
        y = _scaled_gemm(xq, wqt, sx, sw, bias, x.dtype)                  # B operand [N=out, K=in]
        ctx.save_for_backward(xqt, wq, sx, sw)
        ctx.has_bias = bias is not None
        ctx.xshape = x.shape
        return y.reshape(*x.shape[:-1], w.shape[1])

    @staticmethod
    def backward(ctx, dy):
        xqt, wq, sx, sw = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        gq, gqt, sg = quantize_fp8_pair(dy2, torch.float8_e5m2)           # [M, out], [out, M]
        dx = _scaled_gemm(gq, wq, sg, sw, None, dy.dtype).reshape(ctx.xshape)       # dx[M,in] = dy[M,out] @ W^T : B = W [N=in, K=out]
        dw = _scaled_gemm(xqt, gqt, sx, sg, None, dy.dtype)                          # dW[in,out] = x^T[in,M] @ dy[M,out] : B = dy^T [out, M]
        db = dy2.sum(0) if ctx.has_bias else None
        return dx, dw, db


# ------------------------------------------------------------------------------------------------ MX (block-scaled) fp8
def _mx_ok(t):
    return use_fused(t) and t.dim() == 2 and t.dtype in (torch.bfloat16, torch.float16, torch.float32) and t.shape[0] % 128 == 0 and t.shape[1] % 128 == 0


def _mx_sf_index(rows, k, device):
    """Flat byte index of the scale of (row, k-block of 32) inside the 512-byte blocks the block-scaled MMA reads (csrc/quant_fp8.cu)."""
    r = torch.arange(rows, device=device).unsqueeze(1)
    kb = torch.arange(k // 32, device=device).unsqueeze(0)
    return (((r // 128) * (k // 128) + kb // 4) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + kb % 4).reshape(-1)


def quantize_mx(t):
    """OCP MX (microscaling) e4m3 along the last axis of a [rows, K] tensor: one power-of-two scale (E8M0 byte = exponent + 127) per 32
    consecutive elements, rounded up so that no element saturates.  Returns (q [rows, K] e4m3, sf uint8 blocks)."""
    t = raw(t)
    if _mx_ok(t):
        q, sf = ext().quantize_mx(t.contiguous())
        return q, sf
    rows, k = t.shape
    blk = t.float().reshape(rows, k // 32, 32)
    amax = blk.abs().amax(-1)
    e = torch.ceil(torch.log2(amax.clamp_min(1e-38) / E4M3_MAX)).clamp(-127, 127)
    e = torch.where(amax > 0, e, torch.full_like(e, -127.0))
    q = (blk * torch.exp2(-e).unsqueeze(-1)).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn).reshape(rows, k)
    sf = torch.zeros(rows // 128 * (k // 128) * 512, dtype=torch.uint8, device=t.device)
    sf[_mx_sf_index(rows, k, t.device)] = (e + 127).to(torch.uint8).reshape(-1)
    return q, sf


def dequantize_mx(q, sf):
    """fp32 [rows, K] value of an MX-quantised tensor (the reference the block-scaled GEMM is tested against)."""
    q, sf = raw(q), raw(sf)
    if q.is_cuda and use_fused(q):
        return ext().dequantize_mx(q.contiguous(), sf.contiguous())
    rows, k = q.shape
    e = sf[_mx_sf_index(rows, k, q.device)].float().reshape(rows, k // 32) - 127.0
    return (q.float().reshape(rows, k // 32, 32) * torch.exp2(e).unsqueeze(-1)).reshape(rows, k)


def mx_gemm(a, sfa, b, sfb, bias=None, out_dtype=torch.bfloat16):
    """a [M,K], b [N,K] e4m3 with MX scale blocks -> (a * 2^sfa) @ (b * 2^sfb)^T: fp8 wgmma, the scales
    are applied per 32-wide k-block in registers (csrc/gemm_fp8_sm100.cu, MX variant)."""
    a, sfa, b, sfb, bias = raw(a), raw(sfa), raw(b), raw(sfb), raw(bias)
    if use_fused(a) and a.shape[0] % 128 == 0 and b.shape[0] % 128 == 0 and a.shape[1] % 128 == 0:
        bb = bias.to(out_dtype).contiguous() if bias is not None else None
        return ext().gemm_fp8_mx(a.contiguous(), sfa.contiguous(), b.contiguous(), sfb.contiguous(), bb, out_dtype)
    out = dequantize_mx(a, sfa) @ dequantize_mx(b, sfb).t()
    if bias is not None:
        out = out + bias.float()
    return out.to(out_dtype)


class _MxFp8Linear(torch.autograd.Function):
    """y = x @ W (W: [in, out]) with MX block-scaled e4m3 operands in all three GEMMs.  Block scaling runs along the contraction axis, so
    each GEMM quantises its two operands along ITS k: forward k = in, dgrad k = out, wgrad k = tokens."""

    @staticmethod
    def forward(ctx, x, w, bias):
        x2 = x.reshape(-1, x.shape[-1])
        xq, sx = quantize_mx(x2)                               # [M, in] along in
        wq, sw = quantize_mx(w.t().contiguous())               # [out, in] along in
        y = mx_gemm(xq, sx, wq, sw, bias, x.dtype)
        ctx.save_for_backward(x2, w)
        ctx.has_bias = bias is not None
        ctx.xshape = x.shape
        return raw(y).reshape(*x.shape[:-1], w.shape[1])

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        dy2 = dy.reshape(-1, dy.shape[-1]).contiguous()
        gq, sg = quantize_mx(dy2)                              # [M, out] along out
        wq, sw = quantize_mx(w.contiguous())                   # [in, out] along out
        dx = raw(mx_gemm(gq, sg, wq, sw, None, dy.dtype)).reshape(ctx.xshape)
        xtq, sxt = quantize_mx(x2.t().contiguous())            # [in, M] along tokens
        gtq, sgt = quantize_mx(dy2.t().contiguous())           # [out, M] along tokens
        dw = raw(mx_gemm(xtq, sxt, gtq, sgt, None, dy.dtype))
        db = dy2.sum(0) if ctx.has_bias else None
        return dx, dw, db


def mx_fp8_linear(x, weight, bias=None):
    """Linear with MX block-scaled fp8 GEMMs (FLAGS_b200_fp8_block_scaled); shapes that are not multiples of 128 use the per-tensor path."""
    x, weight, bias = raw(x), raw(weight), raw(bias)
    m = x.numel() // x.shape[-1]
    if x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and x.shape[-1] % 128 == 0 and weight.shape[1] % 128 == 0 and m % 128 == 0:
        return wrap(_MxFp8Linear.apply(x, weight, bias))
    return fp8_linear(x, weight, bias)


def fp8_linear(x, weight, bias=None):
    x, weight, bias = raw(x), raw(weight), raw(bias)
    from ..framework.flags import flag

    if flag("FLAGS_b200_fp8_block_scaled", False) and x.is_cuda and x.shape[-1] % 128 == 0 and weight.shape[1] % 128 == 0 and (x.numel() // x.shape[-1]) % 128 == 0 \
            and x.dtype in (torch.bfloat16, torch.float16):
        return wrap(_MxFp8Linear.apply(x, weight, bias))
    if x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and x.shape[-1] % 16 == 0 and weight.shape[1] % 16 == 0 \
            and (x.numel() // x.shape[-1]) % 16 == 0:
        return wrap(_Fp8Linear.apply(x, weight, bias))
    y = torch.matmul(x, weight)
    return wrap(y if bias is None else y + bias)
