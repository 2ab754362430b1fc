"""Device-side MoE routing and the grouped-GEMM expert FFN (csrc/moe.cu, csrc/gemm_sm100.cu grouped modes).

Token slots are laid out grouped by expert in 256-row aligned segments (`moe_route`: counts -> segment starts -> destination row of
every slot, plus the tile -> expert table and the per-expert reduction ranges, all on the device); the expert FFN is then TWO launches
of the persistent wgmma kernel over the stacked expert weights, whatever the number of experts, with no host
synchronisation anywhere (the reference's fused_moe: paddle/phi/kernels/fusion/cutlass/fused_moe_kernel.cu:46, and its gate utility
kernels number_count / assign_pos / limit_by_capacity / prune_gate_by_capacity_kernel.cu:33).

Weight-only int8 / int4 experts (`expert_ffn_weight_only`) use a compact layout instead (`moe_wo_plan`: no padding, a work list of
(expert, token tile) items) for the grouped in-SM dequantising GEMM of csrc/gemm_wo_sm100.cu, or dequantise their stacks for the path above.
"""
from __future__ import annotations

import torch

from . import ext, raw
from . import wgrad as WG


def grouped_ok(x, w1, w2):
    """The grouped wgmma path needs CUDA bf16 / fp16 operands and GEMM dims the kernel accepts."""
    if w1.dtype != x.dtype or w2.dtype != x.dtype or not (w1.is_contiguous() and w2.is_contiguous()):
        return False
    return _grouped_dims_ok(x, w1.shape[1], w1.shape[2], w2.shape[1], w2.shape[2])


def _grouped_dims_ok(x, d, f1, f, d2):
    from ..framework.flags import flag
    from . import use_fused

    if not (use_fused(x) and flag("FLAGS_b200_gemm_backend", "tcgen05") == "tcgen05" and flag("FLAGS_b200_moe_grouped_gemm", True)):
        return False
    return x.dtype in (torch.bfloat16, torch.float16) and all(v >= 256 and v % 8 == 0 for v in (d, f1, f, d2))


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


def _act(h, act):
    from . import activation as KA

    if act == "swiglu":
        return raw(KA.swiglu(h))
    if act == "gelu":
        return torch.nn.functional.gelu(h)
    return torch.relu(h)


def expert_ffn_grouped(x2, expert_idx, weights, w1, w2, act="swiglu"):
    """Top-k MoE FFN over local experts.  x2 [T, d]; expert_idx int64 [T, k] (-1 = dropped); weights [T, k] or None (plain sum);
    w1 [E, d, F1], w2 [E, f, d] stacked.  Returns [T, d].  w1 / w2 may also be zero-argument callables that produce the stack when it is
    needed (the dequantised weights of `expert_ffn_weight_only`: only one of them is alive at a time)."""
    T, k = expert_idx.shape
    w1 = w1() if callable(w1) else w1
    E = w1.shape[0]
    plan = route(expert_idx.reshape(-1), E, rows_cap(T * k, E))
    xp = _Dispatch.apply(x2, plan["dest"], k, plan["cap"])
    h = grouped_linear(xp, w1, plan)
    del w1
    a = _act(h, act)
    y = grouped_linear(a, w2() if callable(w2) else w2, plan)
    return _Combine.apply(y, plan["dest"], weights, k)


# S = tokens x top-k routed slots up to which the weight-only expert FFN runs the in-SM dequantising kernel; larger batches dequantise each
# stack once and run the 16-bit grouped GEMM.  scripts/bench_moe_weight_only.py (DESIGN.md) measured the in-SM route at least as fast as the
# dequantise route at every slot count up to 4096, for Mixtral-8x7B's layer and a 64-expert layer, int8 / int4, per-channel / g128.
WO_MOE_MAX_SLOTS = 4096


def wo_experts_ok(x2, n_expert, k1, n1, k2, n2, group_size):
    """The in-SM weight-only expert kernel takes CUDA bf16 / fp16 rows, fan-ins that are multiples of 64 (and of the scale group) and at
    most 1024 experts (the planning kernel's limit)."""
    from . import use_fused

    if not (use_fused(x2) and x2.dtype in (torch.bfloat16, torch.float16)):
        return False
    g = max(64, group_size)
    return n_expert <= 1024 and k1 % g == 0 and k2 % g == 0 and n1 % 8 == 0 and n2 % 8 == 0


def dequantize_experts(q, s, int4, group_size, dtype):
    """Stacked weight_quantize outputs q [E, N, K] (int4 [E, N, K/2]), fp32 scales [E, N] / [E, K/G, N] -> [E, K, N] in dtype: one kernel on
    CUDA (bf16 / fp16 / fp32), else the torch expression of nn.quant per expert.  Both give the bits of nn.quant.weight_dequantize."""
    if q.is_cuda and dtype in (torch.bfloat16, torch.float16, torch.float32):
        return ext().weight_dequantize_experts(q, s, bool(int4), int(group_size) if group_size > 0 else -1, dtype)
    from ..nn.quant import _dequantize_torch

    return torch.stack([_dequantize_torch(q[e], s[e], int4, dtype, group_size) for e in range(q.shape[0])])


def expert_ffn_weight_only(x2, expert_idx, weights, q1, s1, q2, s2, int4, group_size, b1=None, b2=None, act="swiglu"):
    """Top-k MoE FFN over weight-only int8 / int4 experts (inference).  x2 [T, d]; expert_idx int64 [T, k] (-1 = dropped); weights [T, k]
    fp32 or None; q1 int8 [E, F1, d] (int4 [E, F1, d/2]), q2 [E, d, f] (int4 [E, d, f/2]): stacked weight_quantize outputs; s1 / s2 fp32
    [E, N] or [E, K / group_size, N]; b1 [E, F1] / b2 [E, d] biases in x2's dtype or None.  Returns [T, d].

    S = T * k <= WO_MOE_MAX_SLOTS (known on the host): plan, scatter, two grouped weight-only GEMMs (csrc/gemm_wo_sm100.cu, the int weights
    of the selected experts expanded inside the SM), the activation and the weighted combine - no host read.  Otherwise, and on the CPU:
    each stack is dequantised in one pass when it is needed and the 16-bit code runs unchanged (`expert_ffn_grouped`, or the
    expert-by-expert loop with biases or shapes the grouped GEMM does not take)."""
    T, k = expert_idx.shape
    n1, k1, n2, k2 = q1.shape[1], x2.shape[1], q2.shape[1], q2.shape[2] * (2 if int4 else 1)
    if T * k <= WO_MOE_MAX_SLOTS and wo_experts_ok(x2, q1.shape[0], k1, n1, k2, n2, group_size):
        return expert_ffn_in_sm(x2, expert_idx, weights, q1, s1, q2, s2, int4, group_size, b1, b2, act)
    return expert_ffn_dequantized(x2, expert_idx, weights, q1, s1, q2, s2, int4, group_size, b1, b2, act)


def expert_ffn_in_sm(x2, expert_idx, weights, q1, s1, q2, s2, int4, group_size, b1=None, b2=None, act="swiglu"):
    """The in-SM route of `expert_ffn_weight_only` at any slot count (wo_experts_ok must hold)."""
    T, k = expert_idx.shape
    S, E = T * k, q1.shape[0]
    C = ext()
    gs = int(group_size) if group_size > 0 else -1
    bias = [None if b is None else raw(b).reshape(E, -1).to(x2.dtype).contiguous() for b in (b1, b2)]
    dest, offsets, work = C.moe_wo_plan(expert_idx.reshape(-1).contiguous(), E)
    xp = C.moe_rows_scatter(x2.contiguous(), dest, None, k, S)
    h = C.weight_only_gemm_experts(xp, q1, s1, bias[0], offsets, work, bool(int4), gs)
    y = C.weight_only_gemm_experts(_act(h, act).contiguous(), q2, s2, bias[1], offsets, work, bool(int4), gs)
    return C.moe_rows_combine(y, dest, None if weights is None else weights.reshape(-1).float().contiguous(), k)


def expert_ffn_dequantized(x2, expert_idx, weights, q1, s1, q2, s2, int4, group_size, b1=None, b2=None, act="swiglu"):
    """The dequantise route of `expert_ffn_weight_only`: the 16-bit code on stacks dequantised one at a time."""
    E = q1.shape[0]
    n1, k1, n2, k2 = q1.shape[1], x2.shape[1], q2.shape[1], q2.shape[2] * (2 if int4 else 1)
    deq1 = lambda: dequantize_experts(q1, s1, int4, group_size, x2.dtype)   # noqa: E731
    deq2 = lambda: dequantize_experts(q2, s2, int4, group_size, x2.dtype)   # noqa: E731
    if b1 is None and b2 is None and _grouped_dims_ok(x2, k1, n1, k2, n2):
        return expert_ffn_grouped(x2, expert_idx, weights, deq1, deq2, act)
    from ..incubate.moe import _moe_ffn_loop

    return _moe_ffn_loop(x2, expert_idx, weights, deq1, b1, deq2, b2, act, E)
