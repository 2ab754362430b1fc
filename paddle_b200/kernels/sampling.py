"""Token sampling: one launch samples every row of a [rows, vocab] matrix of logits or probabilities (csrc/sampling.cu).

`sample` runs the sm_90a kernel on CUDA tensors and `sample_ref`, the torch reference with the same definitions, on CPU tensors; the
tests use the reference as the oracle.  Per-row parameters are tensors on x's device, so a CUDA call reads nothing on the host:
temperature (<= 0: greedy), top_k (0: off), top_p (1: off), threshold (optional), seed and offset (int64).

The rules are defined by value, so a row's token depends only on its own values and parameters, never on the other rows:
- greedy: argmax, the lowest index among equal values (torch.argmax's rule);
- top_k: keep every token whose value is >= the k-th largest value, ties included;
- top_p: with w_i = exp(logit_i / T - max) (probabilities: w_i = p_i) over the top-k set and Z = sum w, keep token i when the mass of
  the strictly larger tokens is <= top_p * Z;
- draw: exponential race (Gumbel-max), argmax over the kept tokens of s_i - log(-log u_i), s_i = logit_i / T (probabilities: log p_i);
- threshold: non-truncated, tokens below it (other than the top-1) leave the race; truncated, a winner below it (other than the top-1)
  falls back to the smallest kept token >= threshold (lowest index), or to the top-1 when there is none.
u_i depends only on (seed, offset, i): Philox4x32-10 with key (seed lo, seed hi) and counter (i >> 2, 0, offset lo, offset hi), output
word i & 3, u = ((w >> 8) + 0.5) * 2^-24.  Only where the top-p boundary falls depends on an fp32 sum (the kernel's histogram order).
"""
from __future__ import annotations

import torch

from . import ext, raw

_U32 = 0xFFFFFFFF
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def _mulhilo(a, m):
    """(hi, lo) 32-bit halves of a * m for uint32 values held in int64 tensors, without overflowing int64."""
    p_lo, p_hi = (a & 0xFFFF) * m, (a >> 16) * m                 # both < 2^48
    return (p_hi + (p_lo >> 16)) >> 16, (p_lo + ((p_hi & 0xFFFF) << 16)) & _U32


def philox4x32_10(k0, k1, c0, c1, c2, c3):
    """Philox4x32-10 (Salmon et al., SC'11) on int64 tensors holding uint32 values; returns the four output words."""
    k0, k1, c0, c1, c2, c3 = (torch.as_tensor(t, dtype=torch.int64) for t in (k0, k1, c0, c1, c2, c3))
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _U32, (k1 + _W1) & _U32
        hi0, lo0 = _mulhilo(c0, _M0)
        hi1, lo1 = _mulhilo(c2, _M1)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return c0, c1, c2, c3


def uniforms(seed, offset, n):
    """The race's u_0 .. u_{n-1} for one (seed, offset), float32 [n]."""
    return _uniforms(torch.tensor([int(seed)]), torch.tensor([int(offset)]), n)[0]


def _uniforms(seed, offset, n):
    """u [rows, n] for int64 seed / offset [rows]."""
    seed, offset = seed.reshape(-1, 1).long(), offset.reshape(-1, 1).long()
    i = torch.arange(n, dtype=torch.int64).reshape(1, -1)
    words = torch.stack(philox4x32_10(seed & _U32, (seed >> 32) & _U32, i >> 2, torch.zeros_like(i), offset & _U32, (offset >> 32) & _U32), -1)
    w = words.gather(-1, (i & 3).expand(words.shape[:-1]).unsqueeze(-1)).squeeze(-1)
    return ((w >> 8).float() + 0.5) * 2.0 ** -24


def race_parts(x, temperature, top_k, top_p, seed, offset, threshold=None, is_prob=False, truncated=True):
    """The reference's intermediate values (CPU): ids [rows], race keys [rows, vocab] (-inf outside the race), the top-p mass of the
    strictly larger tokens over Z [rows, vocab] (float64), and masks of the rows that are greedy and that apply top_p."""
    x = raw(x).detach().cpu()
    v = x.float()
    rows, vocab = v.shape
    T = raw(temperature).detach().cpu().float().reshape(rows, 1)
    greedy = ~(T > 0)
    idx = torch.arange(vocab).expand(rows, vocab)
    top1 = v.argmax(-1)
    asc = v.sort(-1).values
    k = raw(top_k).detach().cpu().long().reshape(rows, 1)
    k_on = (k > 0) & (k < vocab) & ~greedy
    kept = ~k_on | (v >= asc.gather(1, vocab - k.clamp(1, vocab)))
    if is_prob:
        s, w = v.log(), v
    else:
        s = v / torch.where(greedy, torch.ones_like(T), T)
        w = torch.exp(s - s.max(-1, keepdim=True).values)
    w = torch.where(kept, w, torch.zeros_like(w)).double()
    z = w.sum(-1, keepdim=True)
    order = torch.sort(v, dim=-1, descending=True, stable=True).indices
    cum = w.gather(1, order).cumsum(-1)
    cex = torch.cat([torch.zeros(rows, 1, dtype=cum.dtype), cum[:, :-1]], 1)
    first = vocab - torch.searchsorted(asc, v, right=True)              # descending position of each value's first occurrence
    above = cex.gather(1, first)
    p = raw(top_p).detach().cpu().float().reshape(rows, 1)
    p_on = (p < 1) & ~greedy
    kept &= ~p_on | (above <= p.double() * z)
    u = _uniforms(raw(seed).detach().cpu(), raw(offset).detach().cpu(), vocab)
    r = s - torch.log(-torch.log(u))
    elig = kept
    thr = None if threshold is None else raw(threshold).detach().cpu().float().reshape(rows, 1)
    if thr is not None and not truncated:
        elig = kept & ((v >= thr) | (idx == top1.reshape(-1, 1)))
    race = torch.where(elig, r, torch.full_like(r, float("-inf")))
    win = race.argmax(-1)
    win = torch.where(race.max(-1).values == float("-inf"), elig.int().argmax(-1), win)
    if thr is not None and truncated:
        ok = kept & (v >= thr)
        fb = torch.where(ok, v, torch.full_like(v, float("inf"))).argmin(-1)
        fb = torch.where(ok.any(-1), fb, top1)
        below = (v.gather(1, win.reshape(-1, 1)).reshape(-1) < thr.reshape(-1)) & (win != top1)
        win = torch.where(below, fb, win)
    ids = torch.where(greedy.reshape(-1), top1, win)
    return ids, race, above / z, greedy.reshape(-1), p_on.reshape(-1)


def sample_ref(x, temperature, top_k, top_p, seed, offset, threshold=None, is_prob=False, truncated=True, k_out=0):
    """The torch reference of `sample` (any device; computed on CPU, returned on x's device)."""
    xr = raw(x)
    ids = race_parts(xr, temperature, top_k, top_p, seed, offset, threshold, is_prob, truncated)[0]
    xc = xr.detach().cpu()
    vals = xc.gather(1, ids.reshape(-1, 1)).reshape(-1)
    k = int(k_out)
    order = torch.sort(xc.float(), dim=-1, descending=True, stable=True).indices[:, :k]   # ties: lowest index first
    dev = xr.device
    return ids.to(dev), vals.to(dev), xc.gather(1, order).to(dev), order.to(dev)


def sample(x, temperature, top_k, top_p, seed, offset, threshold=None, is_prob=False, truncated=True, k_out=0):
    """Samples one token per row of x [rows, vocab] (fp32 / fp16 / bf16 logits, or probabilities with is_prob).  Per-row parameters:
    temperature float32, top_k int32, top_p float32, threshold float32 or None, seed / offset int64, all [rows] on x's device.
    Returns (ids int64 [rows], the chosen values [rows] in x's dtype, the k_out largest values [rows, k_out] and their ids, descending,
    ties by lowest index).  On CUDA this is one kernel launch with no host read."""
    x = raw(x)
    if x.dim() != 2 or x.shape[1] == 0:
        raise ValueError(f"sample: x must be [rows, vocab], got {list(x.shape)}")
    if not 0 <= int(k_out) <= min(1024, x.shape[1]):
        raise ValueError(f"sample: k_out must be in [0, min(1024, vocab)], got {k_out}")
    if x.is_cuda:
        thr = None if threshold is None else raw(threshold)
        return tuple(ext().sample_tokens(x, raw(temperature), raw(top_k), raw(top_p), thr, raw(seed), raw(offset), bool(is_prob),
                                         bool(truncated), int(k_out)))
    return sample_ref(x, temperature, top_k, top_p, seed, offset, threshold, is_prob, truncated, k_out)
