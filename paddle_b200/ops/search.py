"""Search / sort ops. Parity: python/paddle/tensor/search.py."""
from __future__ import annotations

import torch

from ._helpers import T, ax, dt, raw, scalar_or_tensor, to_int, wrap


from ..framework.recording import recordable as _recordable  # noqa: E402

def argmax(x, axis=None, keepdim=False, dtype="int64", name=None):
    x = T(x)
    out = torch.argmax(x, dim=ax(axis), keepdim=keepdim if axis is not None else False)
    if axis is None and keepdim:
        out = out.reshape([1] * x.dim())
    return out.to(dt(dtype))


def argmin(x, axis=None, keepdim=False, dtype="int64", name=None):
    x = T(x)
    out = torch.argmin(x, dim=ax(axis), keepdim=keepdim if axis is not None else False)
    if axis is None and keepdim:
        out = out.reshape([1] * x.dim())
    return out.to(dt(dtype))


def argsort(x, axis=-1, descending=False, stable=False, name=None):
    return torch.argsort(T(x), dim=axis, descending=descending, stable=stable)


def sort(x, axis=-1, descending=False, stable=False, name=None):
    return torch.sort(T(x), dim=axis, descending=descending, stable=stable)[0]


@_recordable
def topk(x, k, axis=None, largest=True, sorted=True, name=None):
    x = T(x)
    v, i = torch.topk(x, int(to_int(k)), dim=-1 if axis is None else axis, largest=largest, sorted=sorted)
    return v, i


def kthvalue(x, k, axis=None, keepdim=False, name=None):
    v, i = torch.kthvalue(T(x), k, dim=-1 if axis is None else axis, keepdim=keepdim)
    return v, i


def mode(x, axis=-1, keepdim=False, name=None):
    v, i = torch.mode(T(x), dim=axis, keepdim=keepdim)
    return v, i


def where(condition, x=None, y=None, name=None):
    c = T(condition)
    if x is None and y is None:
        return tuple(torch.nonzero(c, as_tuple=True))
    return torch.where(c, scalar_or_tensor(x), scalar_or_tensor(y))


def where_(condition, x, y, name=None):
    out = where(condition, x, y)
    with torch.no_grad():
        torch.Tensor.copy_(x, out)
    return x


def nonzero(x, as_tuple=False):
    x = T(x)
    if as_tuple:
        return tuple(i.reshape(-1, 1) for i in torch.nonzero(x, as_tuple=True))
    return torch.nonzero(x)


def searchsorted(sorted_sequence, values, out_int32=False, right=False, name=None):
    return torch.searchsorted(T(sorted_sequence), T(values), out_int32=out_int32, right=right)


def bucketize(x, sorted_sequence, out_int32=False, right=False, name=None):
    return torch.bucketize(T(x), T(sorted_sequence), out_int32=out_int32, right=right)


def index_sample(x, index):
    return torch.gather(T(x), 1, T(index).long())


@_recordable(always=True)                      # a static program draws anew at every run
def top_p_sampling(x, ps, threshold=None, topp_seed=None, seed=-1, k=0, mode="truncated", return_top=False, name=None):
    """Nucleus sampling of one token per row of probabilities x [bs, vocab].  Parity: python/paddle/tensor/search.py:top_p_sampling.

    ps [bs]: each row keeps the tokens whose strictly larger tokens hold at most ps of the mass, and draws among them (kernels.sampling).
    Seeds: topp_seed [bs] gives row b its own seed; else seed >= 0 gives every row that seed, with the row index as the Philox offset;
    seed = -1 takes a seed from the default generator of x's device (advancing it).  threshold [bs]: a token below it is never returned
    unless it is the top-1; mode="truncated" replaces such a draw by the smallest kept token at or above it, "non-truncated" drops the
    tokens below it from the draw.  Returns (values [bs, 1], ids int64 [bs, 1]); with return_top=True and k > 0 also the k largest
    probabilities and their ids [bs, k], descending.  On CUDA the whole call is one kernel launch."""
    from ..kernels.sampling import sample

    x = raw(T(x))
    if x.dim() != 2:
        raise ValueError(f"top_p_sampling: x must be [batch, vocab], got shape {list(x.shape)}")
    if mode not in ("truncated", "non-truncated"):
        raise ValueError(f"top_p_sampling: mode must be 'truncated' or 'non-truncated', got {mode!r}")
    bs, dev = x.shape[0], x.device
    k = int(to_int(k))
    if return_top and not 0 < k <= min(1024, x.shape[1]):
        raise ValueError(f"top_p_sampling: return_top needs 0 < k <= min(1024, vocab), got k={k}")

    def per_row(t, dtype, what):
        t = raw(T(t)).to(dev, dtype).reshape(-1)
        if t.numel() == 1:
            t = t.expand(bs)
        if t.numel() != bs:
            raise ValueError(f"top_p_sampling: {what} needs one value per row ({bs}), got {t.numel()}")
        return t.contiguous()

    top_p = per_row(ps, torch.float32, "ps")
    thr = None if threshold is None else per_row(threshold, torch.float32, "threshold")
    rows = torch.arange(bs, dtype=torch.int64, device=dev)
    if topp_seed is not None:
        seeds, offsets = per_row(topp_seed, torch.int64, "topp_seed"), torch.zeros_like(rows)
    elif seed is not None and int(seed) >= 0:
        seeds, offsets = torch.full_like(rows, int(seed)), rows
    else:
        seeds, offsets = torch.randint(0, 2 ** 62, (1,), dtype=torch.int64, device=dev).expand(bs).contiguous(), rows
    ones = torch.ones(bs, dtype=torch.float32, device=dev)
    no_k = torch.zeros(bs, dtype=torch.int32, device=dev)
    ids, vals, top_vals, top_ids = sample(x, ones, no_k, top_p, seeds, offsets, thr, is_prob=True, truncated=mode == "truncated",
                                          k_out=k if return_top else 0)
    out = (wrap(vals.reshape(bs, 1)), wrap(ids.reshape(bs, 1)))
    return out + (wrap(top_vals), wrap(top_ids)) if return_top else out


__all__ = [n for n in list(globals()) if not n.startswith("_") and n not in ("torch", "T", "ax", "dt", "raw", "scalar_or_tensor", "to_int", "wrap", "annotations")]
