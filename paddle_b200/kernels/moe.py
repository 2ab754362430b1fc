"""Device-side MoE routing and the grouped-GEMM expert FFN (csrc/moe.cu, csrc/gemm_sm100.cu grouped modes).

Token slots are laid out grouped by expert in 256-row aligned segments (`moe_route`: counts -> segment starts -> destination row of
every slot, plus the tile -> expert table and the per-expert reduction ranges, all on the device); the expert FFN is then TWO launches
of the persistent wgmma kernel over the stacked expert weights, whatever the number of experts, with no host
synchronisation anywhere (the reference's fused_moe: paddle/phi/kernels/fusion/cutlass/fused_moe_kernel.cu:46, and its gate utility
kernels number_count / assign_pos / limit_by_capacity / prune_gate_by_capacity_kernel.cu:33).
"""
from __future__ import annotations

import torch

from . import ext, raw
from . import wgrad as WG


def grouped_ok(x, w1, w2):
    """The grouped wgmma path needs CUDA bf16 / fp16 operands and GEMM dims the kernel accepts."""
    from ..framework.flags import flag
    from . import use_fused

    if not (use_fused(x) and flag("FLAGS_b200_gemm_backend", "tcgen05") == "tcgen05" and flag("FLAGS_b200_moe_grouped_gemm", True)):
        return False
    if x.dtype not in (torch.bfloat16, torch.float16) or w1.dtype != x.dtype or w2.dtype != x.dtype:
        return False
    d, f1, f, d2 = w1.shape[1], w1.shape[2], w2.shape[1], w2.shape[2]
    return all(v >= 256 and v % 8 == 0 for v in (d, f1, f, d2)) and w1.is_contiguous() and w2.is_contiguous()


def rows_cap(n_slots, n_expert):
    """Static upper bound of the padded row count (every expert segment rounds up to 256 rows)."""
    return (n_slots + n_expert * 255 + 255) // 256 * 256


def route(expert_idx, n_expert, cap):
    """expert_idx: int64 [S] (-1 = dropped slot). Returns dict(dest, tile_expert, k0, kb, seg, counts) of device tensors."""
    dest, tile_expert, k0, kb, seg, counts = ext().moe_route(expert_idx.contiguous(), int(n_expert), int(cap))
    return dict(dest=dest, tile_expert=tile_expert, k0=k0, kb=kb, seg=seg, counts=counts, cap=int(cap))


class _Dispatch(torch.autograd.Function):
    """xp[dest[i]] = x[i // topk] (rows not addressed stay zero); backward sums the topk rows of every token."""

    @staticmethod
    def forward(ctx, x, dest, topk, cap):
        ctx.save_for_backward(dest)
        ctx.topk = topk
        return ext().moe_rows_scatter(x.contiguous(), dest, None, topk, cap)

    @staticmethod
    def backward(ctx, g):
        (dest,) = ctx.saved_tensors
        return ext().moe_rows_combine(g.contiguous(), dest, None, ctx.topk), None, None, None


class _Combine(torch.autograd.Function):
    """out[t] = sum_k w[t, k] * y[dest[t * topk + k]]."""

    @staticmethod
    def forward(ctx, y, dest, w, topk):
        wf = w.reshape(-1).float().contiguous() if w is not None else None
        ctx.save_for_backward(y, dest, wf if wf is not None else dest)
        ctx.topk, ctx.has_w, ctx.w_dtype, ctx.w_shape = topk, w is not None, (w.dtype if w is not None else None), (w.shape if w is not None else None)
        return ext().moe_rows_combine(y.contiguous(), dest, wf, topk)

    @staticmethod
    def backward(ctx, g):
        y, dest, wf = ctx.saved_tensors
        g = g.contiguous()
        dy = ext().moe_rows_scatter(g, dest, wf if ctx.has_w else None, ctx.topk, y.shape[0])
        dw = None
        if ctx.has_w and ctx.needs_input_grad[2]:
            dw = ext().moe_rows_dot(y, dest, g, ctx.topk).reshape(ctx.w_shape).to(ctx.w_dtype)
        return dy, None, dw, None


class _GroupedLinear(torch.autograd.Function):
    """y[rows of expert e] = xp[rows of expert e] @ w[e]; ONE grouped wgmma launch for all experts."""

    @staticmethod
    def forward(ctx, xp, w, plan_te, plan_k0, plan_kb, sink):
        ctx.save_for_backward(xp, w, plan_te, plan_k0, plan_kb)
        ctx.sink = sink
        return ext().gemm_grouped(xp, w, plan_te, False)

    @staticmethod
    def backward(ctx, dy):
        xp, w, te, k0, kb = ctx.saved_tensors
        dy = dy.contiguous()
        dx = ext().gemm_grouped(dy, w, te, True) if ctx.needs_input_grad[0] else None      # dX = dY W[e]^T (stacked weights read as [N, K])
        dw = None
        if ctx.needs_input_grad[1]:
            sink = ctx.sink
            gbuf = WG._live_gbuf(sink) if sink is not None else None
            if gbuf is not None and not WG.is_deferring():
                ext().gemm_grouped_wgrad(xp, dy, k0, kb, gbuf.view(w.shape))              # accumulate straight into the gradient arena
                WG.stats["fused"] += 1
            else:
                dw = torch.zeros_like(w)
                ext().gemm_grouped_wgrad(xp, dy, k0, kb, dw)
        return dx, dw, None, None, None, None


def grouped_linear(xp, w, plan):
    sink = WG.sink_for(w)
    return _GroupedLinear.apply(xp, raw(w), plan["tile_expert"], plan["k0"], plan["kb"], sink)


def expert_ffn_grouped(x2, expert_idx, weights, w1, w2, act="swiglu"):
    """Top-k MoE FFN over local experts.  x2 [T, d]; expert_idx int64 [T, k] (-1 = dropped); weights [T, k] or None (plain sum);
    w1 [E, d, F1], w2 [E, f, d] stacked.  Returns [T, d]."""
    from . import activation as KA

    T, k = expert_idx.shape
    E = w1.shape[0]
    plan = route(expert_idx.reshape(-1), E, rows_cap(T * k, E))
    xp = _Dispatch.apply(x2, plan["dest"], k, plan["cap"])
    h = grouped_linear(xp, w1, plan)
    if act == "swiglu":
        a = raw(KA.swiglu(h))
    elif act == "gelu":
        a = torch.nn.functional.gelu(h)
    else:
        a = torch.relu(h)
    y = grouped_linear(a, w2, plan)
    return _Combine.apply(y, plan["dest"], weights, k)
