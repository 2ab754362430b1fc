"""GEMM dispatch: wgmma kernel (csrc/gemm_sm100.cu) for bf16/fp16 CUDA operands, torch.matmul otherwise.

``linear(x, W[in,out], b)`` is the framework's Linear primitive with a custom backward that runs all three GEMMs
(y = xW, dx = dy W^T, dW = x^T dy) on the wgmma path without materialising any transpose: the operand "major"
bits of the UMMA descriptors select K-major or MN-major smem tiles.
"""
from __future__ import annotations

import torch

from ..framework.recording import recordable

from . import ext, raw, use_fused, wrap
from ..framework.flags import flag


def _tc_ok(a, b, a_is_km, b_is_nk):
    if not (use_fused(a) and flag("FLAGS_b200_gemm_backend", "tcgen05") == "tcgen05"):
        return False
    if a.dtype not in (torch.bfloat16, torch.float16) or b.dtype != a.dtype:
        return False
    return bool(ext().gemm_supported(a, b, a_is_km, b_is_nk))


def _rowmajor2d(t):
    """2-D view with unit inner stride (copy only if needed)."""
    if t.dim() != 2:
        t = t.reshape(-1, t.shape[-1])
    if t.stride(-1) != 1 or (t.stride(0) % 8 != 0) or (t.data_ptr() % 16 != 0):
        t = t.contiguous()
    return t


def gemm(a, b, bias=None, a_is_km=False, b_is_nk=False, epilogue=0, out=None, out_dtype=None):
    """D = op(A) @ op(B) (+bias, act).  A: [M,K] or [K,M] (a_is_km); B: [K,N] or [N,K] (b_is_nk)."""
    a, b, bias, out = raw(a), raw(b), raw(bias), raw(out)
    if _tc_ok(a, b, a_is_km, b_is_nk):
        ep = epilogue if (epilogue == 4 or bias is not None or epilogue == 0) else epilogue
        if bias is None and epilogue in (1, 2, 3):
            ep = {1: 0, 2: 2, 3: 3}[epilogue]
        return ext().gemm(a, b, bias, a_is_km, b_is_nk, ep, out, out_dtype)
    aa = a.transpose(-1, -2) if a_is_km else a
    bb = b.transpose(-1, -2) if b_is_nk else b
    d = torch.matmul(aa, bb)
    if bias is not None:
        d = d + bias
    if epilogue == 2:
        d = torch.nn.functional.gelu(d)
    elif epilogue == 3:
        d = torch.relu(d)
    if out_dtype is not None:
        d = d.to(out_dtype)
    if out is not None:
        if epilogue == 4:
            out.add_(d)
        else:
            out.copy_(d)
        return out
    return d


class _Linear(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, sink=None):
        x2 = _rowmajor2d(x)
        ctx.save_for_backward(x2, w)
        ctx.x_shape = x.shape
        ctx.has_b = b is not None
        ctx.sink = sink
        # allocate the result in its final shape: a view created inside a custom Function could not be modified in
        # place afterwards (the packed rotary embedding rotates q/k inside the fused QKV output)
        out = torch.empty((*x.shape[:-1], w.shape[1]), dtype=x.dtype, device=x.device)
        ext().gemm(x2, w, b, False, False, 1 if b is not None else 0, out.view(-1, w.shape[1]), None)
        return out

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        dy2 = _rowmajor2d(dy)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            # dx[M,K] = dy[M,N] @ W^T ; W is [K,N] row-major == "[N_out=K, K_red=N]" with the reduction dim contiguous
            dx = ext().gemm(dy2, w, None, False, True, 0, None, None).reshape(ctx.x_shape)
        if ctx.needs_input_grad[1]:
            # dW[K,N] = x^T[K,M] @ dy[M,N] : A = x stored [M,K] -> MN-major A ; B = dy stored [M,N] -> MN-major B
            from . import wgrad as WG

            dw = WG.emit(ctx.sink, x2, dy2)     # fused accumulation into the gradient arena / parked for the pipeline's W pass
        if ctx.has_b and ctx.needs_input_grad[2]:
            db = dy2.sum(0)
        return dx, dw, db, None


class _DeferLinear(torch.autograd.Function):
    """Device-agnostic linear whose weight gradient goes through a wgrad sink (used while a zero-bubble pipeline schedule is
    deferring W passes and the wgmma fast path does not apply, e.g. the CPU/gloo tests or fp32 parameters)."""

    @staticmethod
    def forward(ctx, x, w, b, sink):
        ctx.save_for_backward(x, w)
        ctx.has_b, ctx.sink = b is not None, sink
        y = torch.matmul(x, w)
        return y + b if b is not None else y

    @staticmethod
    def backward(ctx, dy):
        from . import wgrad as WG

        x, w = ctx.saved_tensors
        dy2, x2 = dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1])
        dx = torch.matmul(dy, w.t()) if ctx.needs_input_grad[0] else None
        dw = WG.emit(ctx.sink, x2, dy2) if ctx.needs_input_grad[1] else None
        db = dy2.sum(0) if ctx.has_b and ctx.needs_input_grad[2] else None
        return dx, dw, db, None


@recordable
def linear(x, weight, bias=None):
    from . import wgrad as WG

    weight_in = weight
    x, weight, bias = raw(x), raw(weight), raw(bias)
    if flag("FLAGS_b200_fp8_linear", False) and x.is_cuda and weight.dim() == 2 and weight.dtype == x.dtype:
        from .gemm_fp8 import fp8_linear   # O2-fp8 recipe: e4m3 forward operands, e5m2 output gradients (csrc/gemm_fp8_sm100.cu)

        return fp8_linear(x, weight, bias)
    if x.is_cuda and x.dtype in (torch.bfloat16, torch.float16) and weight.dim() == 2 and weight.dtype == x.dtype \
            and flag("FLAGS_use_fused_kernels", True) and flag("FLAGS_b200_gemm_backend", "tcgen05") == "tcgen05" \
            and x.shape[-1] % 8 == 0 and weight.shape[1] % 8 == 0 and weight.is_contiguous() \
            and (bias is None or bias.dtype == x.dtype) and x.numel() > 0:
        m = x.numel() // x.shape[-1]
        if m % 8 == 0:  # dW needs the token count 16B-aligned for the MN-major map
            return wrap(_Linear.apply(x, weight, bias, WG.sink_for(weight_in)))
    if WG.is_planned() and weight.dim() == 2 and weight.dtype == x.dtype and torch.is_grad_enabled():
        sink = WG.sink_for(weight_in)
        if sink is not None:
            return wrap(_DeferLinear.apply(x, weight, bias, sink))
    from ..amp.auto_cast import fp32_guard

    ctx, (x, weight, bias) = fp32_guard("linear", x, weight, bias)
    with ctx:
        if weight.dim() == 2:
            return wrap(torch.nn.functional.linear(x, weight.t(), bias))   # one addmm; a single autocast unit like the reference's linear op
        y = torch.matmul(x, weight)
        return wrap(y if bias is None else y + bias)


@recordable
def matmul(x, y, transpose_x=False, transpose_y=False):
    """paddle.matmul fast path for 2-D / batched 3-D half-precision operands (no autograd wrapper: used by inference)."""
    x, y = raw(x), raw(y)
    return wrap(gemm(x, y, a_is_km=transpose_x, b_is_nk=transpose_y))
