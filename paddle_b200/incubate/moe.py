"""Mixture-of-Experts. Parity: python/paddle/incubate/distributed/models/moe/{moe_layer,gate/*,utils}.py,
paddle/phi/kernels/gpu/{number_count,assign_pos,limit_by_capacity,prune_gate_by_capacity}_kernel.cu,
paddle/fluid/operators/collective/global_scatter_op.cu.cc / global_gather.

Expert parallelism: tokens are routed top-k, grouped by destination expert, exchanged with ONE all-to-all over the
expert-parallel group (peer-memory kernel csrc/comm/p2p_collectives.cu:alltoall when the symmetric heap is up, NCCL
otherwise), run through the local experts as grouped GEMMs, and combined by the reverse all-to-all.
"""
from __future__ import annotations

import math

import torch
import torch.distributed as dist
import torch.nn.functional as TF

from .. import nn
from ..nn import initializer as I
from ..nn.layer import Layer
from ..tensor import Tensor


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


def _w(t):
    return t.as_subclass(Tensor) if isinstance(t, torch.Tensor) and not isinstance(t, Tensor) else t


# ---- gate utility ops (reference: moe/utils.py) -------------------------------------------------------------------
def _dev_ext(t):
    """The native extension when `t` lives on a GPU (csrc/moe.cu kernels: no host loop, no synchronisation), else None."""
    if isinstance(t, torch.Tensor) and t.is_cuda:
        from .._build import ext

        return ext()
    return None


def _number_count(numbers, upper_range):
    n = _raw(numbers).reshape(-1).long()
    e = _dev_ext(n)
    if e is not None:
        return _w(e.moe_number_count(n.contiguous(), int(upper_range)))
    return _w(torch.bincount(n[n >= 0], minlength=upper_range)[:upper_range])


def _assign_pos(x, cum_count):
    """Positions of tokens grouped by expert id. cum_count = inclusive cumsum of per-expert counts. CPU: stable order; GPU: the
    reference kernel's semantics (assign_pos_kernel.cu: every token claims the next free position of its expert's range)."""
    idx = _raw(x).reshape(-1).long()
    cum = _raw(cum_count).reshape(-1).long()
    e = _dev_ext(idx)
    if e is not None and cum.numel() > 0:
        return _w(e.moe_assign_pos(idx.contiguous(), cum.contiguous(), int(idx.numel())))   # unclaimed tail entries only exist with dropped tokens
    order = torch.argsort(idx[idx >= 0] if bool((idx < 0).any()) else idx, stable=True)
    valid = torch.nonzero(idx >= 0).reshape(-1)
    return _w(valid[order])


def _limit_by_capacity(expert_count, capacity, n_worker):
    ec0, cap0 = _raw(expert_count).reshape(-1).long(), _raw(capacity).reshape(-1).long()
    e = _dev_ext(ec0)
    if e is not None:
        return _w(e.moe_limit_by_capacity(ec0.contiguous(), cap0.contiguous(), int(n_worker)))
    ec = ec0.reshape(n_worker, -1)
    cap = cap0.clone()
    out = torch.zeros_like(ec)
    for w in range(n_worker):
        take = torch.minimum(ec[w], cap)
        out[w] = take
        cap = cap - take
    return _w(out.reshape(-1))


def _prune_gate_by_capacity(gate_idx, expert_count, n_expert, n_worker):
    """Tokens beyond their expert's remaining capacity are dropped (-1).  CPU: arrival order, vectorised (rank of the token within its
    expert via a one-hot cumulative sum); GPU: prune_gate_kernel (atomic countdown like prune_gate_by_capacity_kernel.cu:33)."""
    g = _raw(gate_idx).reshape(-1).long()
    remaining = _raw(expert_count).reshape(-1).long()
    e = _dev_ext(g)
    if e is not None:
        return _w(e.moe_prune_gate_by_capacity(g.contiguous(), remaining.contiguous()))
    valid = g >= 0
    onehot = TF.one_hot(g.clamp(min=0), remaining.numel()) * valid.unsqueeze(-1)
    rank_in_expert = (torch.cumsum(onehot, 0) * onehot).sum(-1)            # 1-based arrival rank inside the token's expert
    keep = valid & (rank_in_expert <= remaining[g.clamp(min=0)])
    return _w(torch.where(keep, g, torch.full_like(g, -1)))


def _random_routing(topk_idx, topk_value, prob, topk=2):
    idx, val = _raw(topk_idx).clone(), _raw(topk_value)
    if topk == 2:
        drop = (2.0 * val[:, 1]) < _raw(prob)
        idx[drop, 1] = -1
    return _w(idx)


number_count, assign_pos, limit_by_capacity, prune_gate_by_capacity, random_routing = _number_count, _assign_pos, _limit_by_capacity, _prune_gate_by_capacity, _random_routing


# ---- all-to-all with autograd -----------------------------------------------------------------------------------------
def _a2a_single(x, in_splits, out_splits, group):
    out = x.new_empty((sum(out_splits), *x.shape[1:]))
    pg = getattr(group, "pg", group)
    if pg is None and not dist.is_initialized():
        return x
    if dist.get_backend(pg) == "gloo":
        n = dist.get_world_size(pg)
        ins = list(x.split(in_splits, 0))
        outs = list(out.split(out_splits, 0))
        me = dist.get_rank(pg)
        for r in range(n):
            gl = dist.get_global_rank(pg, r) if pg is not None else r
            lst = [torch.empty_like(o) for o in outs] if me == r else None
            # gather chunk r of everyone onto rank r
            send = ins[r].contiguous()
            sizes = out_splits if me == r else None
            if me == r:
                lst = [x.new_empty((s, *x.shape[1:])) for s in sizes]
            # variable sizes: pad-free gather via send/recv
            if me == r:
                for j in range(n):
                    if j == r:
                        lst[j].copy_(send)
                    else:
                        dist.recv(lst[j], src=dist.get_global_rank(pg, j) if pg is not None else j, group=pg)
                for o, l in zip(outs, lst):
                    o.copy_(l)
            else:
                dist.send(send, dst=gl, group=pg)
        return out
    dist.all_to_all_single(out, x.contiguous(), out_splits, in_splits, group=pg)
    return out


def _symm_ctx(group, x):
    """Peer-memory context for the expert-parallel group (None -> NCCL path)."""
    if not x.is_cuda or x.dtype not in (torch.bfloat16, torch.float16, torch.float32) or (x.shape[-1] * x.element_size()) % 16:
        return None
    from ..framework.flags import flag

    if not flag("FLAGS_b200_p2p_collectives", True):
        return None
    from ..parallel import symm

    return symm.context_for(group)


class _FusedDispatch(torch.autograd.Function):
    """x[tok] + all-to-all in ONE peer-memory push kernel (csrc/comm/p2p_collectives.cu:a2av_kernel); backward = combine push
    followed by the scatter-add into dx."""

    @staticmethod
    def forward(ctx, x, tok, in_splits, out_splits, sc, cap):
        out = sc.a2av(x, in_splits, sum(out_splits), cap, gather=tok, tag="moe_dispatch")
        ctx.cfg = (in_splits, out_splits, sc, x.shape[0], cap)
        ctx.save_for_backward(tok)
        return out

    @staticmethod
    def backward(ctx, g):
        in_splits, out_splits, sc, n, cap = ctx.cfg
        (tok,) = ctx.saved_tensors
        rows = sc.a2av(g.contiguous(), out_splits, sum(in_splits), cap, tag="moe_combine")
        dx = torch.zeros((n, g.shape[-1]), dtype=g.dtype, device=g.device).index_add_(0, tok, rows)
        return dx, None, None, None, None, None


class _FusedCombine(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, in_splits, out_splits, sc, cap):
        ctx.cfg = (in_splits, out_splits, sc, cap)
        return sc.a2av(y, in_splits, sum(out_splits), cap, tag="moe_combine")

    @staticmethod
    def backward(ctx, g):
        in_splits, out_splits, sc, cap = ctx.cfg
        return sc.a2av(g.contiguous(), out_splits, sum(in_splits), cap, tag="moe_dispatch"), None, None, None, None


class _A2AVDev(torch.autograd.Function):
    """Rows pushed to their destination ranks by the fused gather + all-to-all kernel, split sizes on the device.  backward = the
    reverse push (+ scatter-add into the gathered source rows)."""

    @staticmethod
    def forward(ctx, x, gather, send_rows, recv_rows, sc, cap_out, cap_back, tag):
        ctx.cfg = (sc, cap_back, tag, x.shape[0], gather is not None)
        ctx.save_for_backward(send_rows, recv_rows, gather if gather is not None else send_rows)
        out = sc.a2av_dev(x, send_rows, cap_out, gather=gather, tag=tag + "_f", rows_hint=(gather.numel() if gather is not None else x.shape[0]))
        # dispatch: the consumer copies the rows into the grouped layout at once and keeps nothing -> hand out the symmetric buffer itself;
        # return: the combine keeps its input for the gate-weight gradient, and the buffer is reused by the next layer -> copy ([S, d] only)
        return out if gather is not None else out.clone()

    @staticmethod
    def backward(ctx, g):
        sc, cap_back, tag, n_src, has_gather = ctx.cfg
        send_rows, recv_rows, gather = ctx.saved_tensors
        rows = sc.a2av_dev(g.contiguous(), recv_rows, cap_back, gather=None, tag=tag + "_b", rows_hint=g.shape[0])
        if has_gather:
            dx = torch.zeros((n_src, g.shape[-1]), dtype=g.dtype, device=g.device)
            n = min(rows.shape[0], gather.shape[0])
            # rows beyond what came back are stale: they belong to dropped slots, whose sorted position is past every valid one
            valid = (torch.arange(n, device=g.device) < send_rows.sum()).unsqueeze(-1)
            dx.index_add_(0, gather[:n], torch.where(valid, rows[:n], torch.zeros_like(rows[:n])))
            return dx, None, None, None, None, None, None, None
        return rows.clone(), None, None, None, None, None, None, None


class _EPExperts(torch.autograd.Function):
    """dispatch push -> grouped expert FFN -> return push, as one differentiable unit built from differentiable pieces."""

    @staticmethod
    def forward(ctx, *a):
        raise RuntimeError("use _EPExperts.apply")

    @classmethod
    def apply(cls, x, tok_sorted, send_rows, recv_rows, row_e, w1, w2, layer, sc, cap, S):
        from ..kernels import moe as KM

        xs = _A2AVDev.apply(x, tok_sorted, send_rows, recv_rows, sc, cap, S, "moe_ep_dispatch")          # [cap, d], rows of my experts
        plan = KM.route(row_e, layer.num_expert, KM.rows_cap(cap, layer.num_expert))
        xp = KM._Dispatch.apply(xs, plan["dest"], 1, plan["cap"])
        h = KM.grouped_linear(xp, layer.experts.w1, plan)
        from ..kernels import activation as KA

        act = layer.experts.activation
        a = _raw(KA.swiglu(h)) if act == "swiglu" else (TF.gelu(h) if act == "gelu" else torch.relu(h))
        y = KM.grouped_linear(a, layer.experts.w2, plan)
        ys = KM._Combine.apply(y, plan["dest"], None, 1)                                                  # back in arrival order [cap, d]
        return _A2AVDev.apply(ys, None, recv_rows, send_rows, sc, S, cap, "moe_ep_return")               # [S, d] in my sorted-slot order


class _AllToAll(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, in_splits, out_splits, group):
        ctx.cfg = (in_splits, out_splits, group)
        return _a2a_single(x, in_splits, out_splits, group)

    @staticmethod
    def backward(ctx, g):
        in_splits, out_splits, group = ctx.cfg
        return _a2a_single(g.contiguous(), out_splits, in_splits, group), None, None, None


def global_scatter(x, local_count, global_count, group=None, use_calc_stream=True):
    """Send rows of x (sorted by destination expert) to the ranks owning those experts. Parity: moe/utils.py:global_scatter."""
    lc, gc = _raw(local_count).reshape(-1), _raw(global_count).reshape(-1)
    world = _world(group)
    n_exp = lc.numel() // world
    in_splits = lc.reshape(world, n_exp).sum(1).tolist()
    out_splits = gc.reshape(world, n_exp).sum(1).tolist()
    return _w(_AllToAll.apply(_raw(x), in_splits, out_splits, group))


def global_gather(x, local_count, global_count, group=None, use_calc_stream=True):
    lc, gc = _raw(local_count).reshape(-1), _raw(global_count).reshape(-1)
    world = _world(group)
    n_exp = lc.numel() // world
    in_splits = gc.reshape(world, n_exp).sum(1).tolist()
    out_splits = lc.reshape(world, n_exp).sum(1).tolist()
    return _w(_AllToAll.apply(_raw(x), in_splits, out_splits, group))


def _world(group):
    if group is None:
        return dist.get_world_size() if dist.is_initialized() else 1
    return group.nranks if hasattr(group, "nranks") else dist.get_world_size(group)


def _rank(group):
    if group is None:
        return dist.get_rank() if dist.is_initialized() else 0
    return group.rank if hasattr(group, "nranks") else dist.get_rank(group)


# ---- gates ----------------------------------------------------------------------------------------------------------------
class BaseGate(Layer):
    def __init__(self, num_expert, world_size):
        super().__init__()
        self.world_size, self.num_expert = world_size, num_expert
        self.tot_expert = world_size * num_expert
        self.loss = None

    def set_loss(self, loss):
        self.loss = loss

    def get_loss(self, clear=True):
        l = self.loss
        if clear:
            self.loss = None
        return l


class NaiveGate(BaseGate):
    def __init__(self, d_model, num_expert, world_size, topk=2):
        super().__init__(num_expert, world_size)
        self.gate = nn.Linear(d_model, self.tot_expert)
        self.top_k = topk

    def forward(self, inp, return_all_scores=False):
        gate = self.gate(inp)
        val, idx = torch.topk(_raw(gate), self.top_k, -1)
        return (_w(val), _w(idx), gate) if return_all_scores else (_w(val), _w(idx))


class GShardGate(NaiveGate):
    def __init__(self, d_model, num_expert, world_size, topk=2, capacity=(1.2, 2.4), random_routing=True, group=None):
        super().__init__(d_model, num_expert, world_size, topk)
        self.capacity, self.random_routing, self.group = capacity, random_routing, group

    def forward(self, x):
        val, idx, gate = super().forward(x, return_all_scores=True)
        score = TF.softmax(_raw(gate).float(), -1)
        s = score.shape[0]
        top1 = _raw(idx)[:, 0]
        c_e = torch.bincount(top1, minlength=self.tot_expert).float() / s
        m_e = score.mean(0)
        self.set_loss(_w((c_e * m_e).mean() * (self.num_expert ** 2)))
        cap_rate = self.capacity[0 if self.training else 1]
        capacity = math.ceil(cap_rate * s)
        cnt = torch.zeros(self.tot_expert, dtype=torch.long, device=top1.device)
        idx2 = _raw(idx).clone()
        flat = idx2.reshape(-1)
        # capacity pruning in arrival order (vectorised rank-within-expert)
        onehot = TF.one_hot(flat.clamp(min=0), self.tot_expert)
        pos = (torch.cumsum(onehot, 0) * onehot).sum(-1)
        flat[pos > capacity] = -1
        idx2 = flat.reshape(idx2.shape)
        if self.random_routing and self.training and self.top_k == 2:
            idx2 = _raw(_random_routing(idx2, torch.softmax(_raw(val).float(), -1), torch.rand(s, device=top1.device)))
        return val, _w(idx2)


class SwitchGate(NaiveGate):
    def __init__(self, d_model, num_expert, world_size, topk=1, switch_eps=0.1, capacity=(1.2, 2.4), group=None):
        super().__init__(d_model, num_expert, world_size, topk=1)
        self.switch_eps, self.capacity, self.group = switch_eps, capacity, group

    def forward(self, inp):
        score = _raw(self.gate(inp))
        if self.training:
            score = score + (torch.rand_like(score) * 2 * self.switch_eps + 1.0 - self.switch_eps).log()
        p = TF.softmax(score.float(), -1)
        val, idx = p.max(-1, keepdim=True)
        s = p.shape[0]
        cap = math.ceil(self.capacity[0 if self.training else 1] * s / self.tot_expert)
        onehot = TF.one_hot(idx[:, 0], self.tot_expert)
        pos = (torch.cumsum(onehot, 0) * onehot).sum(-1)
        idx = idx.clone()
        idx[pos > cap, 0] = -1
        frac = onehot.float().mean(0)
        self.set_loss(_w((frac * p.mean(0)).sum() * self.tot_expert))
        return _w(val.to(inp.dtype)), _w(idx)


# ---- expert FFN (grouped) ------------------------------------------------------------------------------------------------
def _expert_ffn(x, counts, w1, b1, w2, b2, act):
    """x rows sorted by local expert; counts[e] rows per expert; w1 [E, d, f(or 2f)], w2 [E, f, d].  w1 / w2 may be zero-argument
    callables that produce the stack (dequantised experts): every expert's first layer runs before the second stack is made."""
    from ..kernels import activation as KA
    from ..kernels import gemm as KG

    w1 = w1() if callable(w1) else w1
    hs, off = [], 0
    for e, c in enumerate(counts):
        xe = x[off:off + c]
        off += c
        if c == 0:
            hs.append(None)
            continue
        h = _raw(KG.linear(xe, w1[e], None if b1 is None else b1[e]))
        if act == "swiglu":
            h = _raw(KA.swiglu(h))
        else:
            h = TF.gelu(h) if act == "gelu" else torch.relu(h)
        hs.append(h)
    del w1
    w2 = w2() if callable(w2) else w2
    outs = [x.new_zeros((0, w2.shape[-1])) if h is None else _raw(KG.linear(h, w2[e], None if b2 is None else b2[e])) for e, h in enumerate(hs)]
    return torch.cat(outs, 0) if outs else x.new_zeros((0, w2.shape[-1]))


def _moe_ffn_loop(x2, idx, val, w1, b1, w2, b2, act, n_expert):
    """out[t] = sum_k val[t, k] * expert_{idx[t, k]}(x2[t]) with the experts run one after another over the rows sorted by expert
    (slots with idx -1 are dropped; val None: plain sum)."""
    flat_e = idx.reshape(-1)
    tok = torch.arange(x2.shape[0], device=x2.device).repeat_interleave(idx.shape[-1])
    wv = val.reshape(-1) if val is not None else torch.ones(flat_e.shape, device=x2.device)
    keep = flat_e >= 0
    flat_e, tok, wv = flat_e[keep], tok[keep], wv[keep]
    order = torch.argsort(flat_e, stable=True)
    tok = tok[order]
    counts = torch.bincount(flat_e, minlength=n_expert).tolist()
    y = _expert_ffn(x2[tok], counts, w1, b1, w2, b2, act)
    w = wv[order].to(y.dtype)
    return torch.zeros_like(x2).index_add(0, tok, y * w[:, None])


_QUANT_METHODS = {"None": None, "weight_only_int8": False, "weight_only_int4": True}   # -> int4


def _quantized_stack(w, scale, int4, n_expert, k, name):
    """(q int8 [E, N, K] (int4 [E, N, K/2]), scale fp32, group_size) of a stack of weight_quantize outputs of n_expert experts with fan-in
    k; N comes from the scale ([E, N] per-channel, [E, K / G, N] with G = 64 / 128).  Any view holding the same bytes (e.g. [E, K, N]) is
    accepted."""
    q, s = _raw(w), _raw(scale)
    gs = -1
    if s.dim() == 3 and s.shape[1] > 0 and k % s.shape[1] == 0 and k // s.shape[1] in (64, 128):
        gs = k // s.shape[1]
    if (s.dim() != 2 and gs < 0) or s.shape[0] != n_expert:
        raise ValueError(f"{name}: scale of shape {tuple(s.shape)} is neither [E, N] (per-channel) nor [E, K / G, N] with E = {n_expert}, "
                         f"K = {k} and G 64 or 128")
    E, N = s.shape[0], s.shape[-1]
    if q.dtype != torch.int8 or (int4 and k % 2) or q.numel() != E * N * (k // 2 if int4 else k):
        raise ValueError(f"{name}: expected the int8 bytes of {E} experts x {N} outputs x {k} inputs{' (int4: two per byte)' if int4 else ''}, "
                         f"got {q.dtype} of shape {tuple(q.shape)}")
    return q.contiguous().reshape(E, N, k // 2 if int4 else k), s.float().contiguous(), gs


def moe_ffn(x, gate_weight, ffn1_weight, ffn1_bias, ffn2_weight, ffn2_bias, topk=2, norm_topk_prob=True, ffn1_scale=None, ffn2_scale=None,
            quant_method="None"):
    """Single-device fused MoE (all experts local). x [.., d]; ffn1 [E, d, 2f] (swiglu) ; ffn2 [E, f, d].  quant_method
    "weight_only_int8" / "weight_only_int4": the ffn weights hold the bytes of stacked `weight_quantize` outputs ([E, N, K], int4
    [E, N, K/2]) and ffn*_scale their scales ([E, N] or [E, K / G, N]); they run through kernels.moe.expert_ffn_weight_only."""
    if quant_method not in _QUANT_METHODS:
        raise ValueError(f"quant_method must be one of {sorted(_QUANT_METHODS)}, got {quant_method!r}")
    int4 = _QUANT_METHODS[quant_method]
    if int4 is None and (ffn1_scale is not None or ffn2_scale is not None):
        raise ValueError('ffn1_scale / ffn2_scale are only used with a weight-only quant_method, not "None"')
    if int4 is None and (_raw(ffn1_weight).dtype == torch.int8 or _raw(ffn2_weight).dtype == torch.int8):
        raise ValueError('int8 expert weights need quant_method "weight_only_int8" or "weight_only_int4" and their scales')
    if int4 is not None and (ffn1_scale is None or ffn2_scale is None):
        raise ValueError(f"quant_method {quant_method!r} needs ffn1_scale and ffn2_scale")
    xr = _raw(x)
    shape = xr.shape
    x2 = xr.reshape(-1, shape[-1])
    logits = x2.float() @ _raw(gate_weight).float()
    p = torch.softmax(logits, -1)
    val, idx = p.topk(topk, -1)
    if norm_topk_prob:
        val = val / val.sum(-1, keepdim=True)
    from ..kernels import moe as KM

    if int4 is not None:
        d, E = shape[-1], _raw(gate_weight).shape[-1]
        f = _raw(ffn2_weight).numel() * (2 if int4 else 1) // (E * d)   # ffn2's fan-in, from its byte count
        q1, s1, gs1 = _quantized_stack(ffn1_weight, ffn1_scale, int4, E, d, "ffn1")
        q2, s2, gs2 = _quantized_stack(ffn2_weight, ffn2_scale, int4, E, f, "ffn2")
        if s2.shape[-1] != d or gs1 != gs2 or q1.shape[1] not in (f, 2 * f):
            raise ValueError(f"ffn1 {tuple(q1.shape)} / ffn2 {tuple(q2.shape)} quantised experts do not form [E, d = {d}, 2f or f] -> [E, f, d] "
                             "with one scale layout")
        act = "swiglu" if q1.shape[1] == 2 * f else "gelu"
        b1 = None if ffn1_bias is None else _raw(ffn1_bias)
        b2 = None if ffn2_bias is None else _raw(ffn2_bias)
        out = KM.expert_ffn_weight_only(x2, idx, val.to(torch.float32), q1, s1, q2, s2, int4, gs1, b1, b2, act)
        return _w(out.reshape(shape))
    E = _raw(ffn1_weight).shape[0]
    if KM.grouped_ok(x2, _raw(ffn1_weight), _raw(ffn2_weight)) and ffn1_bias is None and ffn2_bias is None:
        act_g = "swiglu" if _raw(ffn1_weight).shape[-1] == 2 * _raw(ffn2_weight).shape[1] else "gelu"
        out = KM.expert_ffn_grouped(x2, idx, val.to(torch.float32), ffn1_weight, ffn2_weight, act_g)   # grouped tcgen05 GEMMs, routing on the device
        return _w(out.reshape(shape))
    act = "swiglu" if _raw(ffn1_weight).shape[-1] == 2 * _raw(ffn2_weight).shape[1] else "gelu"
    out = _moe_ffn_loop(x2, idx, val, _raw(ffn1_weight), None if ffn1_bias is None else _raw(ffn1_bias), _raw(ffn2_weight),
                        None if ffn2_bias is None else _raw(ffn2_bias), act, E)
    return _w(out.reshape(shape))


class ExpertFFN(Layer):
    """num_expert local SwiGLU (or GELU) FFN experts stored as stacked weights [E, ...] (grouped GEMM friendly)."""

    def __init__(self, num_expert, d_model, d_hidden, activation="swiglu"):
        super().__init__()
        self.num_expert, self.activation = num_expert, activation
        f1 = 2 * d_hidden if activation == "swiglu" else d_hidden
        self.w1 = self.create_parameter([num_expert, d_model, f1], default_initializer=I.Normal(0.0, 0.02))
        self.w2 = self.create_parameter([num_expert, d_hidden, d_model], default_initializer=I.Normal(0.0, 0.02))
        for p in (self.w1, self.w2):
            p.no_sync = True   # expert parameters are not data-parallel replicated across the expert group

    def forward(self, x, counts):
        return _w(_expert_ffn(_raw(x), counts, _raw(self.w1), None, _raw(self.w2), None, self.activation))


class WeightOnlyExpertFFN(Layer):
    """The experts of an `ExpertFFN` with weight-only int8 / int4 weights (inference).  Every expert's [in, out] weight goes through
    nn.quant.weight_quantize: `quant_w1` int8 [E, F1, d] (int4 [E, F1, d/2]) and `quant_w2` [E, d, f] (int4 [E, d, f/2]) with fp32 scales
    `scale_w1` / `scale_w2` ([E, N] per-channel or [E, K / group_size, N]).  They are buffers, as in WeightOnlyLinear: the layer has nothing
    to train.  MoELayer runs it through kernels.moe.expert_ffn_weight_only."""

    def __init__(self, experts, algo="weight_only_int8", group_size=-1):
        super().__init__()
        from ..nn import quant as Q

        self.num_expert, self.activation = experts.num_expert, experts.activation
        self.algo, self.group_size, self.int4 = algo, int(group_size), algo == "weight_only_int4"
        for name in ("w1", "w2"):
            w = _raw(getattr(experts, name)).detach().float()
            qs = [Q.weight_quantize(w[e].as_subclass(Tensor), algo=algo, group_size=self.group_size) for e in range(w.shape[0])]
            self.register_buffer("quant_" + name, torch.stack([_raw(q) for q, _ in qs]))
            self.register_buffer("scale_" + name, torch.stack([_raw(s).float() for _, s in qs]).contiguous())

    def dequantized(self, dtype):
        """(w1 [E, d, F1], w2 [E, f, d]) in `dtype`: the 16-bit stacks this layer computes with, bit-equal to weight_dequantize per expert."""
        from ..kernels import moe as KM

        return tuple(KM.dequantize_experts(getattr(self, "quant_" + n), getattr(self, "scale_" + n), self.int4, self.group_size, dtype)
                     for n in ("w1", "w2"))

    def ffn(self, x, idx, probs):
        """Top-k expert FFN of rows x [T, d] routed to idx [T, k] with weights probs [T, k] (kernels.moe.expert_ffn_weight_only)."""
        from ..kernels import moe as KM

        return KM.expert_ffn_weight_only(x, idx, probs, self.quant_w1, self.scale_w1, self.quant_w2, self.scale_w2, self.int4, self.group_size,
                                         act=self.activation)

    def forward(self, x, counts):
        from ..kernels import moe as KM

        xr = _raw(x)
        deq = lambda n: (lambda: KM.dequantize_experts(getattr(self, "quant_" + n), getattr(self, "scale_" + n), self.int4,   # noqa: E731
                                                       self.group_size, xr.dtype))
        return _w(_expert_ffn(xr, counts, deq("w1"), None, deq("w2"), None, self.activation))

    def extra_repr(self):
        g = "per-channel" if self.group_size <= 0 else f"group_size={self.group_size}"
        return f"num_expert={self.num_expert}, {self.algo}, {g}"


class MoELayer(Layer):
    """Parity: python/paddle/incubate/distributed/models/moe/moe_layer.py:MoELayer.

    experts: a LayerList of per-expert Layers (reference style) or an ExpertFFN (stacked, fast path).
    gate: dict(type='gshard'|'switch'|'naive', top_k=..) or a BaseGate instance. moe_group: expert-parallel group.
    """

    def __init__(self, d_model, experts, gate=None, moe_group=None, mp_group=None, recompute_interval=0, recompute_ctx=None,
                 ep_capacity_factor=2.0):
        super().__init__()
        self.d_model, self.group = d_model, moe_group
        self.ep_capacity_factor = float(ep_capacity_factor)   # device-side expert-parallel path: receive capacity = factor x local slots
        self.world_size = _world(moe_group) if (moe_group is not None or dist.is_initialized()) else 1
        if moe_group is None:
            self.world_size = 1
        self.experts = experts
        self.num_expert = experts.num_expert if isinstance(experts, (ExpertFFN, WeightOnlyExpertFFN)) else len(experts)
        gate = gate or {"type": "gshard", "top_k": 2}
        if isinstance(gate, dict):
            k = gate.get("top_k", 2)
            t = gate.get("type", "gshard")
            if t == "naive" or t is None:
                gate = NaiveGate(d_model, self.num_expert, self.world_size, topk=k)
            elif t == "gshard":
                gate = GShardGate(d_model, self.num_expert, self.world_size, topk=k, group=moe_group)
            elif t == "switch":
                gate = SwitchGate(d_model, self.num_expert, self.world_size, topk=k, group=moe_group)
            else:
                raise ValueError(f"unknown gate type {t}")
        self.gate = gate
        self.top_k = gate.top_k

    def forward(self, inp):
        xr = _raw(inp)
        shape = xr.shape
        x = xr.reshape(-1, shape[-1])
        val, idx = self.gate(_w(x))
        val, idx = _raw(val), _raw(idx)
        k = idx.shape[-1]
        probs = torch.softmax(val.float(), -1) if not isinstance(self.gate, SwitchGate) else val.float()
        from ..kernels import moe as KM

        if isinstance(self.experts, WeightOnlyExpertFFN) and self.world_size == 1:
            return _w(self.experts.ffn(x, idx.long(), probs).reshape(shape))
        grouped = isinstance(self.experts, ExpertFFN) and KM.grouped_ok(x, _raw(self.experts.w1), _raw(self.experts.w2))
        if grouped and self.world_size == 1:
            out = KM.expert_ffn_grouped(x, idx.long(), probs, self.experts.w1, self.experts.w2, self.experts.activation)
            return _w(out.reshape(shape))
        if grouped and self.world_size > 1:
            out = self._forward_ep_device(x, idx.long(), probs)
            if out is not None:
                return _w(out.reshape(shape))
        flat_e = idx.reshape(-1)
        keep = flat_e >= 0
        tok_all = torch.arange(x.shape[0], device=x.device).repeat_interleave(k)
        fe, tok, w = flat_e[keep], tok_all[keep], probs.reshape(-1)[keep]
        order = torch.argsort(fe, stable=True)
        fe, tok, w = fe[order], tok[order], w[order]
        tot = self.num_expert * self.world_size
        local_count = torch.bincount(fe, minlength=tot)
        if self.world_size > 1:
            global_count = torch.empty_like(local_count)
            pg = getattr(self.group, "pg", self.group)
            if dist.get_backend(pg) == "gloo":
                lst = [torch.empty_like(local_count) for _ in range(self.world_size)]
                dist.all_gather(lst, local_count, group=pg)
                me = _rank(self.group)
                global_count = torch.cat([l.reshape(self.world_size, self.num_expert)[me] for l in lst])
            else:
                dist.all_to_all_single(global_count, local_count, group=pg)
            sc = _symm_ctx(self.group, x)
            ins = local_count.reshape(self.world_size, self.num_expert).sum(1).tolist()
            outs = global_count.reshape(self.world_size, self.num_expert).sum(1).tolist()
            cap = sc.a2av_capacity(sum(ins), sum(outs), x) if sc is not None else 0
            fused = cap > 0
            if fused:   # gather + dispatch in one kernel, rows land directly in the expert ranks' HBM over NVLink
                xs = _FusedDispatch.apply(x, tok, ins, outs, sc, cap)
            else:
                xs = _raw(global_scatter(x[tok], local_count, global_count, self.group))
            # received rows are ordered (src rank, local expert): regroup by local expert
            gc = global_count.reshape(self.world_size, self.num_expert)
            seg_e = torch.arange(self.num_expert, device=x.device).repeat(self.world_size)
            row_e = torch.repeat_interleave(seg_e, gc.reshape(-1))
            perm = torch.argsort(row_e, stable=True)
            counts = gc.sum(0).tolist()
            y = self._run_experts(xs[perm], counts)
            inv = torch.empty_like(perm)
            inv[perm] = torch.arange(perm.numel(), device=perm.device)
            if fused:
                y = _FusedCombine.apply(y[inv].contiguous(), outs, ins, sc, cap)
            else:
                y = _raw(global_gather(y[inv], local_count, global_count, self.group))
        else:
            y = self._run_experts(x[tok], local_count.tolist())
        out = torch.zeros_like(x).index_add(0, tok, y * w[:, None].to(y.dtype))
        return _w(out.reshape(shape))

    def _forward_ep_device(self, x, idx, probs):
        """Expert parallelism with every decision on the device: slots are sorted by destination, the per-(rank, expert) counts are
        exchanged with a tiny peer-memory all-to-all, rows travel with the fused gather + all-to-all push kernel (split sizes read from
        device memory), the local experts run as grouped tcgen05 GEMMs over a device-built plan, and the reverse push + a weighted
        top-k combine finish the layer.  No .item() / .tolist() / NCCL call anywhere."""
        from ..kernels import moe as KM

        sc = _symm_ctx(self.group, x)
        if sc is None:
            return None
        W, El = self.world_size, self.num_expert
        T, k = idx.shape
        S, d = T * k, x.shape[-1]
        tot = W * El
        # static receive capacity: every source rank sends at most C slots to any one expert (slots beyond that are dropped, the
        # usual capacity rule of GShard / Switch routing), so a rank receives at most W * El * C = ep_capacity_factor * S rows
        cf = float(getattr(self, "ep_capacity_factor", 2.0))
        C = max(1, math.ceil(cf * S / tot))
        cap = (W * El * C + 255) // 256 * 256
        need = (cap + S) * d * x.element_size() + (64 << 20)
        if need > sc.heap.size() - sc._base_cursor:
            return None
        flat_e = _raw(_prune_gate_by_capacity(idx.reshape(-1), torch.full((tot,), C, dtype=torch.int64, device=x.device), tot, 1))
        key = torch.where(flat_e >= 0, flat_e, torch.full_like(flat_e, tot))
        order = torch.argsort(key, stable=True)                        # slots grouped by destination rank (then expert); dropped slots last
        tok_sorted = torch.div(order, k, rounding_mode="floor")
        local_count = _raw(_number_count(flat_e, tot)).reshape(W, El)  # what this rank sends, per (rank, expert)
        global_count = sc.exchange_counts(local_count, tag="moe_counts")   # [src rank, local expert]: what arrives here
        send_rows, recv_rows = local_count.sum(1), global_count.sum(1)
        inv = torch.empty_like(order)
        inv[order] = torch.arange(S, device=x.device)
        dest_back = torch.where(flat_e >= 0, inv, torch.full_like(inv, -1)).to(torch.int32)   # slot -> row of the returned buffer
        # rows received from (src rank, local expert) segments -> local expert id per row (-1 beyond what arrived)
        bounds = torch.cumsum(global_count.reshape(-1), 0)
        seg = torch.bucketize(torch.arange(cap, device=x.device), bounds, right=True)
        row_e = torch.where(seg < tot, seg % El, torch.full_like(seg, -1))
        y_back = _EPExperts.apply(x, tok_sorted, send_rows, recv_rows, row_e, _raw(self.experts.w1), _raw(self.experts.w2), self, sc, cap, S)
        return KM._Combine.apply(y_back, dest_back, probs, k)

    def _run_experts(self, x, counts):
        if isinstance(self.experts, (ExpertFFN, WeightOnlyExpertFFN)):
            return _raw(self.experts(x, counts))
        outs, off = [], 0
        for e, c in enumerate(counts):
            xe = x[off:off + c]
            off += c
            outs.append(_raw(self.experts[e](_w(xe))) if c > 0 else xe.new_zeros((0, self.d_model)))
        return torch.cat(outs, 0)


class ClipGradForMOEByGlobalNorm:
    """Global-norm clip where expert params' norms are summed over the moe group. Parity: moe/grad_clip.py."""

    def __init__(self, clip_norm, is_expert_param_func=None, moe_group=None, group_name="default_moe_group"):
        self.clip_norm, self.is_expert, self.group = float(clip_norm), is_expert_param_func or (lambda p: getattr(p, "no_sync", False)), moe_group

    def __call__(self, params_grads):
        sq_n = sq_e = None
        for p, g in params_grads:
            if g is None:
                continue
            s = _raw(g).float().pow(2).sum()
            if self.is_expert(p):
                sq_e = s if sq_e is None else sq_e + s
            else:
                sq_n = s if sq_n is None else sq_n + s
        dev = next((g.device for _, g in params_grads if g is not None), "cpu")
        z = torch.zeros((), device=dev)
        sq_e = z if sq_e is None else sq_e
        if self.group is not None and _world(self.group) > 1:
            sq_e = sq_e.reshape(1).clone()
            dist.all_reduce(sq_e, group=getattr(self.group, "pg", self.group))
            sq_e = sq_e.reshape([])
        total = torch.sqrt((z if sq_n is None else sq_n) + sq_e)
        coef = self.clip_norm / torch.clamp(total, min=self.clip_norm)
        return [(p, g if g is None else g * coef.to(g.dtype)) for p, g in params_grads]
