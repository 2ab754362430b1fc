"""Attention entry point ([B,S,H,D] layout). Parity: paddle flash_attention / scaled_dot_product_attention
(python/paddle/nn/functional/flash_attention.py).

Dispatch: the sm_90a wgmma flash kernels for fp16/bf16, head_dim 128 (csrc/attention_sm100.cu) or 64
(csrc/attention_d64_sm100.cu), no explicit mask — they read q/k/v in place as strided views of a packed QKV
projection, and a column-wise row-range mask (attention_colmask) runs on the same kernels.  Attention dropout (0 < p < 1) runs on
their dropout instantiations (csrc/attention_dropout_sm100.cu): the mask is a pure function of (seed, offset, batch, head, query,
key) (dropout_keep_mask is its torch twin), drawn from torch's CUDA generator or a given `seed_offset` (int64 [2]), and the backward
regenerates it from the pair the forward used.  Column-masked calls run kernels that skip the tiles the mask hides and leave out the
per-element mask test where it hides nothing (csrc/attention_flashmask_sm100.cu; colmask_tile_classes is the torch twin of their tile
classes); B200_ATTN_MASK_SKIP=0 sends them to the kernels that test every element instead, for comparison.  Other head sizes, dense
masks and dropout >= 1 take the PyTorch SDPA (library) path.  Backward: csrc/attention_bwd_sm100.cu (B200_ATTN_BWD=own, default) or, for comparison, a library backward
fed with our forward's (out, logsumexp) (B200_ATTN_BWD=cudnn|flash).  The own backward is a single pass that bulk-reduces dQ in
arrival order (reproducible to rounding); FLAGS_cudnn_deterministic switches it to a bitwise-reproducible dK/dV + dQ kernel pair.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from ..framework.flags import flag
from ..framework.recording import recordable
from . import ext, raw, use_fused, wrap


def attention_ref(q, k, v, mask=None, dropout_p=0.0, causal=False, scale=None):
    b, sq, h, d = q.shape
    hk = k.shape[2]
    qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
    if hk != h:
        rep = h // hk
        kt = kt.repeat_interleave(rep, 1)
        vt = vt.repeat_interleave(rep, 1)
    if mask is not None and mask.dtype != torch.bool and mask.dtype != q.dtype:
        mask = mask.to(q.dtype)
    out = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=mask, dropout_p=dropout_p, is_causal=causal and mask is None, scale=scale)
    return out.transpose(1, 2)


_bwd_backend = [__import__("os").environ.get("B200_ATTN_BWD", "own")]   # own | cudnn | flash
# column-masked calls: True: the tile-skipping kernels; False (B200_ATTN_MASK_SKIP=0): the kernels that test every element
_mask_skip = [__import__("os").environ.get("B200_ATTN_MASK_SKIP", "1") != "0"]


_U32 = 0xFFFFFFFF


def dropout_keep(p):
    """The kernels' 16-bit keep threshold: an element is kept iff its draw is below round((1 - p) * 2^16)."""
    return int(round((1.0 - float(p)) * 65536.0))


def dropout_keep_mask(seed, offset, b, h, sq, sk, p=0.1, device=None):
    """The attention dropout mask of the kernels, bool [b, h, sq, sk] (True: kept), for a call with generator (seed, offset).

    Element (b, h, i, j) is kept iff its 16-bit Philox4x32-10 draw is below dropout_keep(p) (csrc/include/b200_philox.cuh): key
    (seed lo, seed hi), counter (kc, rc, (offset + b H + h) lo, hi) with rc = 8 (i >> 4) + (i & 7), kc = 4 (j >> 4) + ((j & 7) >> 1),
    half (j & 1) of output word 2 ((i >> 3) & 1) + ((j >> 3) & 1).  Computed on the CPU with int64 torch ops."""
    from .sampling import philox4x32_10

    seed, offset = int(seed) & 0xFFFFFFFFFFFFFFFF, int(offset)
    i = torch.arange(sq, dtype=torch.int64)
    j = torch.arange(sk, dtype=torch.int64)
    rc = ((i >> 4) << 3) | (i & 7)                                         # [sq]
    kc = ((j >> 4) << 2) | ((j & 7) >> 1)                                  # [sk]
    plane = offset + torch.arange(b * h, dtype=torch.int64)                # [b h]
    nr, nk = int(rc.max()) + 1 if sq else 0, int(kc.max()) + 1 if sk else 0
    P, R, C = torch.meshgrid(torch.arange(b * h), torch.arange(nr), torch.arange(nk), indexing="ij")
    words = torch.stack(philox4x32_10(seed & _U32, (seed >> 32) & _U32, C, R, plane[P] & _U32, (plane[P] >> 32) & _U32), -1).reshape(-1)
    word = 2 * ((i >> 3) & 1).reshape(-1, 1) + ((j >> 3) & 1).reshape(1, -1)                      # [sq, sk]
    at = ((torch.arange(b * h).reshape(-1, 1, 1) * nr + rc.reshape(1, -1, 1)) * nk + kc.reshape(1, 1, -1)) * 4 + word
    draw = (words[at] >> (16 * (j & 1))) & 0xFFFF
    keep = (draw < dropout_keep(p)).reshape(b, h, sq, sk)
    return keep.to(device) if device is not None else keep


def _seed_offset_arg(seed_offset):
    """fixed seed_offset (paddle's fixed_seed_offset: int64 [2] = (seed, offset)) as a tensor the kernels read, or None."""
    if seed_offset is None:
        return None
    t = raw(seed_offset)
    if not isinstance(t, torch.Tensor):
        t = torch.tensor([int(x) for x in t], dtype=torch.int64)
    return t.to(torch.int64).reshape(2).contiguous()


def _dropout_ok(dropout_p):
    return 0.0 <= float(dropout_p) < 1.0


class _FlashAttn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale, causal, dropout_p=0.0, seed_offset=None):
        res = ext().attention_fwd(q, k, v, scale, causal, False, None, dropout_p, seed_offset)
        out, lse = res[0], res[1]
        so = res[2] if dropout_p > 0.0 else None
        ctx.save_for_backward(q, k, v, out, lse, so)
        ctx.scale, ctx.causal, ctx.dropout_p = scale, causal, dropout_p
        ctx.seed_offset = so
        if so is not None:
            ctx.mark_non_differentiable(so)
        return out, so

    @staticmethod
    def backward(ctx, do, _dso=None):
        q, k, v, out, lse, so = ctx.saved_tensors
        do = do.contiguous()
        if ctx.dropout_p > 0.0:
            dq, dk, dv = ext().attention_bwd(q, k, v, out, lse, do, ctx.scale, ctx.causal, None, ctx.dropout_p, so)
            return dq, dk, dv, None, None, None, None
        if _bwd_backend[0] == "own":   # csrc/attention_bwd_sm100.cu: single pass, or dK/dV + dQ kernels under FLAGS_cudnn_deterministic
            dq, dk, dv = ext().attention_bwd(q, k, v, out, lse, do, ctx.scale, ctx.causal)
            return dq, dk, dv, None, None, None, None
        if _bwd_backend[0] == "cudnn" and q.shape[2] == k.shape[2]:
            # Hopper-tuned library backward fed with OUR forward's (out, logsumexp); [B,S,H,D] tensors enter as [B,H,S,D] views
            try:
                z = torch.zeros((), dtype=torch.int64, device=q.device)
                dq, dk, dv = torch.ops.aten._scaled_dot_product_cudnn_attention_backward(
                    do.transpose(1, 2), q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), out.transpose(1, 2), lse.unsqueeze(-1), z, z,
                    None, None, None, q.shape[1], k.shape[1], 0.0, ctx.causal, scale=ctx.scale)
                return dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2), None, None, None, None
            except Exception:  # noqa: BLE001  (op unavailable / shape unsupported: use the flash backward from here on)
                _bwd_backend[0] = "flash"
        empty = torch.empty(0, dtype=torch.int64, device=q.device)
        rng = torch.zeros(2, dtype=torch.int64, device=q.device)
        dq, dk, dv = torch.ops.aten._flash_attention_backward(do, q, k, v, out, lse, None, None, q.shape[1], k.shape[1], 0.0, ctx.causal,
                                                               rng, empty, scale=ctx.scale)
        return dq, dk, dv, None, None, None, None


class _FlashAttnColMask(torch.autograd.Function):
    """wgmma flash attention with a column-wise row-range mask (flashmask / packed variable-length sequences / sliding windows):
    colmask int32 [B, 1|H, Sk, 4] = (lt_start, lt_end, ut_start, ut_end): key j hides query rows [lt_start, lt_end) and
    [ut_start, ut_end).  Forward and backward are the same kernels as the dense path (csrc/attention_sm100.cu,
    attention_bwd_sm100.cu) with the mask test added to their score-tile loops."""

    @staticmethod
    def forward(ctx, q, k, v, colmask, scale, causal, dropout_p=0.0, seed_offset=None):
        skip = _mask_skip[0]
        res = ext().attention_fwd(q, k, v, scale, causal, False, colmask, dropout_p, seed_offset, skip)
        out, lse = res[0], res[1]
        so = res[2] if dropout_p > 0.0 else None
        ctx.save_for_backward(q, k, v, out, lse, colmask, so)
        ctx.scale, ctx.causal, ctx.dropout_p, ctx.skip = scale, causal, dropout_p, skip
        if so is not None:
            ctx.mark_non_differentiable(so)
        return out, so

    @staticmethod
    def backward(ctx, do, _dso=None):
        q, k, v, out, lse, colmask, so = ctx.saved_tensors
        dq, dk, dv = ext().attention_bwd(q, k, v, out, lse, do.contiguous(), ctx.scale, ctx.causal, colmask, ctx.dropout_p, so, ctx.skip)
        return dq, dk, dv, None, None, None, None, None


_INT_MAX = 2 ** 31 - 1


def colmask_from_startend(startend_row_indices, causal, sq):
    """Paddle flashmask `startend_row_indices` [B, Hm, Sk, {1,2,4}] -> the kernels' int4 form [B, Hm, Sk, 4]."""
    idx = raw(startend_row_indices).to(torch.int32)
    n = idx.shape[-1]
    zero = torch.zeros_like(idx[..., 0])
    big = torch.full_like(zero, _INT_MAX)
    if causal:
        lts, lte = idx[..., 0], (idx[..., 1] if n >= 2 else big)
        uts = ute = zero
    elif n == 1:
        lts, lte, uts, ute = idx[..., 0], big, zero, zero
    elif n == 2:
        lts, lte, uts, ute = idx[..., 0], big, zero, idx[..., 1]
    else:
        lts, lte, uts, ute = idx[..., 0], idx[..., 1], idx[..., 2], idx[..., 3]
    return torch.stack([lts, lte, uts, ute], -1).contiguous()


def colmask_from_cu_seqlens(cu_q, cu_k, total_k, causal=False):
    """Packed variable-length batch -> document mask: key j of sequence s is visible to the query rows [cu_q[s], cu_q[s+1]) only.
    causal: also the causal mask within each sequence, bottom-right aligned like the kernels' causal flag (local query i of a sequence
    of len_q queries and len_k keys sees local key kj iff kj <= i + len_k - len_q), for q and k packed differently; run it with
    causal=False."""
    cu_q, cu_k = raw(cu_q).to(torch.int64), raw(cu_k).to(torch.int64)
    keys = torch.arange(total_k, device=cu_k.device)
    seq = torch.bucketize(keys, cu_k[1:], right=True).clamp(max=cu_q.numel() - 2)
    qs, qe = cu_q[seq].to(torch.int32), cu_q[seq + 1].to(torch.int32)
    valid = keys < cu_k[-1]
    zero = torch.zeros_like(qs)
    lts = torch.where(valid, qe, zero)                          # rows >= qe hidden; keys beyond the last sequence hide every row
    lte = torch.full_like(qs, _INT_MAX)
    if causal:                                                  # rows < qs + max(0, kj - (len_k - len_q)) hidden
        kj = keys - cu_k[seq]
        shift = (cu_k[seq + 1] - cu_k[seq]) - (cu_q[seq + 1] - cu_q[seq])
        qs = qs + (kj - shift).clamp(min=0).to(torch.int32)
    ute = torch.where(valid, qs, zero)                          # rows < qs hidden
    return torch.stack([lts, lte, zero, ute], -1).reshape(1, 1, total_k, 4).contiguous()


def colmask_from_window(sq, sk, left, right, causal, device):
    """Sliding window: query i sees keys in [i - left, i + right] (right = 0 under a causal mask)."""
    keys = torch.arange(sk, device=device, dtype=torch.int32)
    off = sk - sq
    lts = (keys - off + left + 1).clamp(min=0)                  # rows i with key < i + off - left  <=>  i > key - off + left
    lte = torch.full_like(keys, _INT_MAX)
    uts = torch.zeros_like(keys)
    ute = (keys - off - (0 if causal else right)).clamp(min=0) if not causal else torch.zeros_like(keys)   # rows i < key - off - right
    return torch.stack([lts, lte, uts, ute], -1).reshape(1, 1, sk, 4).contiguous()


def attention_colmask(q, k, v, colmask, causal=False, scale=None, dropout_p=0.0, seed_offset=None, return_seed_offset=False):
    """[B,S,H,D] attention under a column-wise row-range mask on the own wgmma kernels; None if the operands do not qualify.
    dropout_p > 0: attention dropout (mask of `seed_offset`, or of torch's CUDA generator); with return_seed_offset the result is
    (out, the int64 [2] (seed, offset) of the mask)."""
    q, k, v = raw(q), raw(k), raw(v)
    if not fused_ok(q, k, v, None, dropout_p, causal):
        return None
    sc = float(scale) if scale is not None else 1.0 / math.sqrt(q.shape[-1])
    out, so = _FlashAttnColMask.apply(q, k, v, raw(colmask).to(torch.int32).contiguous(), sc, bool(causal), float(dropout_p),
                                      _seed_offset_arg(seed_offset))
    return (wrap(out), so) if return_seed_offset else wrap(out)


def colmask_tile_classes(colmask, sq, sk, bm, bn, causal):
    """The tile classes of the tile-skipping kernels, int8 [B, Hm, ceil(sq / bm), ceil(sk / bn)], for query tiles of bm rows against
    key tiles of bn keys: 0 hidden (every key of the tile hides every row of the query tile, or the tile is past the causal limit of the
    query tile's last row: not computed), 1 partial (the per-element mask test runs), 2 open (no key hides a row: no mask test).
    From the min / max of each bound over the tile's keys below sk (csrc/include/b200_mask_tiles.cuh); the kernels use bn = 128 (bm = 128
    in the forward and the deterministic dQ, 64 in dK / dV).  Shapes only: valid without a GPU."""
    m = raw(colmask).long()[..., :sk, :]
    b, hm = m.shape[0], m.shape[1]
    nm, nn = -(-sq // bm), -(-sk // bn)
    pad = nn * bn - sk
    big = torch.iinfo(torch.int64).max

    def ext_(fill, red):
        x = torch.nn.functional.pad(m, (0, 0, 0, pad), value=fill).reshape(b, hm, nn, bn, 4)
        return (x.amax(3) if red == "max" else x.amin(3)).unsqueeze(2)         # [b, hm, 1, nn, 4]
    mx, mn = ext_(-big, "max"), ext_(big, "min")
    r0 = (torch.arange(nm, device=m.device) * bm).reshape(1, 1, nm, 1)
    r1 = r0 + bm
    hidden = ((mx[..., 0] <= r0) & (mn[..., 1] >= r1)) | ((mx[..., 2] <= r0) & (mn[..., 3] >= r1))
    open_ = ((mn[..., 0] >= r1) | (mx[..., 1] <= r0)) & ((mn[..., 2] >= r1) | (mx[..., 3] <= r0))
    cls = torch.where(hidden, 0, torch.where(open_, 2, 1))
    if causal:
        n0 = (torch.arange(nn, device=m.device) * bn).reshape(1, 1, 1, nn)
        cls = torch.where(n0 <= r0 + bm - 1 + (sk - sq), cls, 0)
    return cls.to(torch.int8)


def colmask_to_dense(colmask, sq):
    """Boolean visibility [B, Hm, Sq, Sk] of an int4 column mask (reference path / tests)."""
    m = raw(colmask).long()
    rows = torch.arange(sq, device=m.device).reshape(1, 1, sq, 1)
    lts, lte, uts, ute = (m[..., i].unsqueeze(2) for i in range(4))
    hidden = ((rows >= lts) & (rows < lte)) | ((rows >= uts) & (rows < ute))
    return ~hidden


class _FlashAttnPacked(torch.autograd.Function):
    """Attention over a packed projection qkv [B,S,nh+2*nkv,D] (or [S,B,...] when seq_major): the kernels read q/k/v in place
    through strided TMA maps and the backward writes d(qkv) in place (dk/dv slices straight from the kernel epilogue), so
    autograd never builds zero-filled slice gradients and the sequence-parallel layout needs no transpose copies."""

    @staticmethod
    def forward(ctx, qkv, nh, nkv, scale, causal, seq_major, dropout_p=0.0, seed_offset=None, colmask=None):
        x = qkv.transpose(0, 1) if seq_major else qkv
        q, k, v = x[:, :, :nh], x[:, :, nh:nh + nkv], x[:, :, nh + nkv:]
        skip = _mask_skip[0]
        res = ext().attention_fwd(q, k, v, scale, causal, seq_major, colmask, dropout_p, seed_offset, skip)    # out: same memory order as qkv
        out, lse = res[0], res[1]
        so = res[2] if dropout_p > 0.0 else None
        ctx.save_for_backward(qkv, out, lse, so, colmask)
        ctx.cfg = (nh, nkv, scale, causal, seq_major, dropout_p, skip)
        if so is not None:
            ctx.mark_non_differentiable(so)
        return out, so

    @staticmethod
    def backward(ctx, do, _dso=None):
        qkv, out, lse, so, colmask = ctx.saved_tensors
        nh, nkv, scale, causal, seq_major, dropout_p, skip = ctx.cfg
        if dropout_p > 0.0 or colmask is not None:
            dqkv = ext().attention_bwd_packed(qkv, nh, nkv, out, lse, do.contiguous(), scale, causal, seq_major, dropout_p, so, colmask, skip)
        else:
            dqkv = ext().attention_bwd_packed(qkv, nh, nkv, out, lse, do.contiguous(), scale, causal, seq_major)
        return dqkv, None, None, None, None, None, None, None, None


def attention_packed(qkv, nh, nkv, causal=True, scale=None, seq_major=False, dropout_p=0.0, seed_offset=None, return_seed_offset=False,
                     colmask=None):
    """qkv: [B,S,nh+2*nkv,D] contiguous (q heads | k heads | v heads), or [S,B,...] with seq_major=True (the layout of
    sequence-parallel layers). Returns [B,S,nh,D] (resp. [S,B,nh,D]).  dropout_p, seed_offset, return_seed_offset: as `attention`.
    colmask: int32 [B, 1|nh, S, 4] column mask over the [B,S] view, as attention_colmask; the backward still writes d(qkv) in place.
    Where the kernels do not apply, the reference attention runs with colmask_to_dense."""
    x = raw(qkv)
    xb = x.transpose(0, 1) if seq_major else x
    q, k, v = xb[:, :, :nh], xb[:, :, nh:nh + nkv], xb[:, :, nh + nkv:]
    cm = raw(colmask).to(torch.int32).contiguous() if colmask is not None else None
    if _bwd_backend[0] == "own" and x.is_contiguous() and fused_ok(q, k, v, None, dropout_p, causal):
        sc = float(scale) if scale is not None else 1.0 / math.sqrt(x.shape[-1])
        out, so = _FlashAttnPacked.apply(x, int(nh), int(nkv), sc, bool(causal), bool(seq_major), float(dropout_p), _seed_offset_arg(seed_offset),
                                         cm)
        return (wrap(out), so) if return_seed_offset else wrap(out)
    if return_seed_offset:
        raise ValueError("attention_packed: return_seed_offset needs the own kernels (fp16/bf16, head_dim 64 or 128, 0 <= dropout_p < 1)")
    out = attention(q, k, v, colmask_to_dense(cm, q.shape[1]) if cm is not None else None, dropout_p, causal, scale)
    return wrap(raw(out).transpose(0, 1).contiguous()) if seq_major else out


def fused_ok(q, k, v, mask, dropout_p, causal):
    if not (use_fused(q) and flag("FLAGS_b200_flash_attention", True)) or mask is not None or not _dropout_ok(dropout_p):
        return False
    if q.dtype not in (torch.float16, torch.bfloat16) or q.dim() != 4 or q.shape[-1] not in (64, 128):
        return False
    if causal and q.shape[1] != k.shape[1]:
        return False
    return bool(ext().attention_supported(q, k, v))


@recordable
def attention(q, k, v, mask=None, dropout_p=0.0, causal=False, scale=None, seed_offset=None, return_seed_offset=False):
    """[B,S,H,D] attention.  0 < dropout_p < 1 on the own kernels drops attention probabilities with the mask of `seed_offset` (int64 [2]
    (seed, offset), used as given) or of torch's CUDA generator; return_seed_offset=True returns (out, the pair the mask was drawn
    with), which replays the mask through `seed_offset` and `dropout_keep_mask`."""
    q, k, v, mask = raw(q), raw(k), raw(v), raw(mask)
    if fused_ok(q, k, v, mask, dropout_p, causal):
        sc = float(scale) if scale is not None else 1.0 / math.sqrt(q.shape[-1])
        out, so = _FlashAttn.apply(q, k, v, sc, bool(causal), float(dropout_p), _seed_offset_arg(seed_offset))
        return (wrap(out), so) if return_seed_offset else wrap(out)
    if return_seed_offset:
        raise ValueError("attention: return_seed_offset needs the own kernels (fp16/bf16, head_dim 64 or 128, no dense mask, 0 <= dropout_p < 1)")
    if causal and mask is not None:
        sq, sk = q.shape[1], k.shape[1]
        cm = torch.ones(sq, sk, dtype=torch.bool, device=q.device).tril(sk - sq)
        mask = (mask & cm) if mask.dtype == torch.bool else mask.masked_fill(~cm, float("-inf"))
        causal = False
    return wrap(attention_ref(q, k, v, mask, dropout_p, causal, scale))
