"""Weight-gradient sinks: fused accumulation into the flat gradient arena and deferred ("W pass") execution.

Two things the reference gets from separate mechanisms live here:

* **fused accumulation** (role of ``fused_linear_param_grad_add``, /root/reference/paddle/phi/kernels/fusion/gpu/
  fused_linear_param_grad_add_kernel.cu): when a parameter's gradient is a view of a flat arena slab
  (``parallel/arena.py``) the wgrad GEMM adds straight into it through the accumulate epilogue of the wgmma kernel,
  so no per-micro-batch ``dW`` tensor is allocated and autograd's in-place ``grad += dW`` kernel disappears.
* **deferral** (zero-bubble pipeline schedules, /root/reference/python/paddle/distributed/passes/
  pipeline_scheduler_pass/pipeline_zero_bubble.py:62): inside ``deferring(queue)`` the backward of every linear only
  computes the input gradient (the "B" pass) and parks ``(x, dy)``; ``flush(queue)`` later runs the parked weight
  gradient GEMMs (the "W" pass) wherever the schedule has a bubble to fill.

A sink is only handed out when nobody observes the gradient through autograd hooks (DataParallel / sharding register
post-accumulate hooks on parameters: those keep the classic path).
"""
from __future__ import annotations

import contextlib

import torch

from ..framework.flags import flag

_defer_stack = []     # innermost active queue (list) or nothing
stats = {"parked": 0, "fused": 0, "returned": 0}   # counters for tests / profiling
_planned = [0]        # >0 while a schedule that will defer W passes is running its forwards (see `planning`)


class Sink:
    __slots__ = ("param", "gbuf")

    def __init__(self, param, gbuf):
        self.param, self.gbuf = param, gbuf


def _has_hooks(p):
    bh = getattr(p, "_backward_hooks", None)
    ph = getattr(p, "_post_accumulate_grad_hooks", None)
    return bool(bh) or bool(ph)


def sink_for(weight):
    """Sink for `weight` (a leaf parameter), or None when the ordinary autograd return path must be used."""
    if not isinstance(weight, torch.Tensor) or not weight.requires_grad or not weight.is_leaf:
        return None
    if not flag("FLAGS_b200_fused_wgrad", True) or _has_hooks(weight):
        return None
    gbuf = weight.__dict__.get("_arena_grad") if hasattr(weight, "__dict__") else None
    if gbuf is not None and gbuf.dtype != weight.dtype:
        gbuf = None
    if gbuf is None and not (_defer_stack or _planned[0]):
        return None
    return Sink(weight, gbuf)


def _live_gbuf(sink):
    """The arena view, provided it still IS the parameter's .grad (clear_grad(set_to_zero=False) or a user assignment unhooks it)."""
    g = sink.gbuf
    if g is None:
        return None
    cur = torch.Tensor.grad.__get__(sink.param)
    return g if (cur is not None and cur.data_ptr() == g.data_ptr()) else None


def is_deferring():
    return bool(_defer_stack)


def is_planned():
    return _planned[0] > 0


@contextlib.contextmanager
def planning():
    """Forward passes run inside this context build linears whose weight gradient can be parked later (any device)."""
    _planned[0] += 1
    try:
        yield
    finally:
        _planned[0] -= 1


@contextlib.contextmanager
def deferring(queue):
    """Backward passes run inside this context park their weight-gradient GEMMs in `queue` (a list)."""
    _defer_stack.append(queue)
    try:
        yield queue
    finally:
        _defer_stack.pop()


def _gemm_tn(x2, dy2, out=None):
    """dW[K,N] = x2[M,K]^T @ dy2[M,N] (accumulating into `out` when given)."""
    from . import gemm as KG

    if out is not None:
        return KG.gemm(x2, dy2, a_is_km=True, epilogue=4, out=out)
    return KG.gemm(x2, dy2, a_is_km=True)


def _apply(sink, x2, dy2):
    g = _live_gbuf(sink)
    if g is not None:
        _gemm_tn(x2, dy2, out=g.view(x2.shape[1], dy2.shape[1]))
        return
    dw = _gemm_tn(x2, dy2).reshape(sink.param.shape)
    p = sink.param
    cur = torch.Tensor.grad.__get__(p)
    if cur is None:
        torch.Tensor.grad.__set__(p, dw)
    else:
        cur.add_(dw)


def emit(sink, x2, dy2):
    """Called from a linear's backward. Returns dW for autograd, or None when the sink consumed (or parked) it."""
    if sink is None:
        return _gemm_tn(x2, dy2)
    if _defer_stack:
        _defer_stack[-1].append((sink, x2, dy2))
        stats["parked"] += 1
        return None
    if _live_gbuf(sink) is not None:
        _apply(sink, x2, dy2)
        stats["fused"] += 1
        return None
    stats["returned"] += 1
    return _gemm_tn(x2, dy2)


@torch.no_grad()
def flush(queue, limit=None):
    """Run (up to `limit`) parked weight-gradient GEMMs of `queue`, oldest first. Returns the number executed."""
    n = 0
    while queue and (limit is None or n < limit):
        sink, x2, dy2 = queue.pop(0)
        _apply(sink, x2, dy2)
        n += 1
    return n
