"""Attention entry point ([B,S,H,D] layout). Parity: paddle flash_attention / scaled_dot_product_attention
(python/paddle/nn/functional/flash_attention.py).

Dispatch: the sm_90a wgmma flash kernel (csrc/attention_sm100.cu) for fp16/bf16, head_dim 128, no explicit mask and no
dropout — it reads q/k/v in place as strided views of a packed QKV projection; everything else takes the PyTorch SDPA
(library) path.  Backward: csrc/attention_bwd_sm100.cu (B200_ATTN_BWD=own, default) or, for comparison, a library backward
fed with our forward's (out, logsumexp) (B200_ATTN_BWD=cudnn|flash).
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


class _FlashAttn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, scale, causal):
        out, lse = ext().attention_fwd(q, k, v, scale, causal)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.scale, ctx.causal = scale, causal
        return out

    @staticmethod
    def backward(ctx, do):
        q, k, v, out, lse = ctx.saved_tensors
        do = do.contiguous()
        if _bwd_backend[0] == "own":   # csrc/attention_bwd_sm100.cu: wgmma dK/dV kernel + dQ kernel, no atomics
            dq, dk, dv = ext().attention_bwd(q, k, v, out, lse, do, ctx.scale, ctx.causal)
            return dq, dk, dv, None, None
        if _bwd_backend[0] == "cudnn" and q.shape[2] == k.shape[2]:
            # Hopper-tuned library backward fed with OUR forward's (out, logsumexp); [B,S,H,D] tensors enter as [B,H,S,D] views
            try:
                z = torch.zeros((), dtype=torch.int64, device=q.device)
                dq, dk, dv = torch.ops.aten._scaled_dot_product_cudnn_attention_backward(
                    do.transpose(1, 2), q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), out.transpose(1, 2), lse.unsqueeze(-1), z, z,
                    None, None, None, q.shape[1], k.shape[1], 0.0, ctx.causal, scale=ctx.scale)
                return dq.transpose(1, 2), dk.transpose(1, 2), dv.transpose(1, 2), None, None
            except Exception:  # noqa: BLE001  (op unavailable / shape unsupported: use the flash backward from here on)
                _bwd_backend[0] = "flash"
        empty = torch.empty(0, dtype=torch.int64, device=q.device)
        rng = torch.zeros(2, dtype=torch.int64, device=q.device)
        dq, dk, dv = torch.ops.aten._flash_attention_backward(do, q, k, v, out, lse, None, None, q.shape[1], k.shape[1], 0.0, ctx.causal,
                                                               rng, empty, scale=ctx.scale)
        return dq, dk, dv, None, None


class _FlashAttnColMask(torch.autograd.Function):
    """wgmma flash attention with a column-wise row-range mask (flashmask / packed variable-length sequences / sliding windows):
    colmask int32 [B, 1|H, Sk, 4] = (lt_start, lt_end, ut_start, ut_end): key j hides query rows [lt_start, lt_end) and
    [ut_start, ut_end).  Forward and backward are the same kernels as the dense path (csrc/attention_sm100.cu,
    attention_bwd_sm100.cu) with the mask test added to their score-tile loops."""

    @staticmethod
    def forward(ctx, q, k, v, colmask, scale, causal):
        out, lse = ext().attention_fwd(q, k, v, scale, causal, False, colmask)
        ctx.save_for_backward(q, k, v, out, lse, colmask)
        ctx.scale, ctx.causal = scale, causal
        return out

    @staticmethod
    def backward(ctx, do):
        q, k, v, out, lse, colmask = ctx.saved_tensors
        dq, dk, dv = ext().attention_bwd(q, k, v, out, lse, do.contiguous(), ctx.scale, ctx.causal, colmask)
        return dq, dk, dv, None, None, None


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


def colmask_from_cu_seqlens(cu_q, cu_k, total_k):
    """Packed variable-length batch -> document mask: key j of sequence s is visible to the query rows [cu_q[s], cu_q[s+1]) only."""
    cu_q, cu_k = raw(cu_q).to(torch.int64), raw(cu_k).to(torch.int64)
    keys = torch.arange(total_k, device=cu_k.device)
    seq = torch.bucketize(keys, cu_k[1:], right=True).clamp(max=cu_q.numel() - 2)
    qs, qe = cu_q[seq].to(torch.int32), cu_q[seq + 1].to(torch.int32)
    valid = keys < cu_k[-1]
    zero = torch.zeros_like(qs)
    lts = torch.where(valid, qe, zero)                          # rows >= qe hidden; keys beyond the last sequence hide every row
    lte = torch.full_like(qs, _INT_MAX)
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


def attention_colmask(q, k, v, colmask, causal=False, scale=None):
    """[B,S,H,D] attention under a column-wise row-range mask on the own wgmma kernels; None if the operands do not qualify."""
    q, k, v = raw(q), raw(k), raw(v)
    if not fused_ok(q, k, v, None, 0.0, causal):
        return None
    sc = float(scale) if scale is not None else 1.0 / math.sqrt(q.shape[-1])
    return wrap(_FlashAttnColMask.apply(q, k, v, raw(colmask).to(torch.int32).contiguous(), sc, bool(causal)))


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
    def forward(ctx, qkv, nh, nkv, scale, causal, seq_major):
        x = qkv.transpose(0, 1) if seq_major else qkv
        q, k, v = x[:, :, :nh], x[:, :, nh:nh + nkv], x[:, :, nh + nkv:]
        out, lse = ext().attention_fwd(q, k, v, scale, causal, seq_major)    # out: same memory order as qkv
        ctx.save_for_backward(qkv, out, lse)
        ctx.cfg = (nh, nkv, scale, causal, seq_major)
        return out

    @staticmethod
    def backward(ctx, do):
        qkv, out, lse = ctx.saved_tensors
        nh, nkv, scale, causal, seq_major = ctx.cfg
        return ext().attention_bwd_packed(qkv, nh, nkv, out, lse, do.contiguous(), scale, causal, seq_major), None, None, None, None, None


def attention_packed(qkv, nh, nkv, causal=True, scale=None, seq_major=False):
    """qkv: [B,S,nh+2*nkv,D] contiguous (q heads | k heads | v heads), or [S,B,...] with seq_major=True (the layout of
    sequence-parallel layers). Returns [B,S,nh,D] (resp. [S,B,nh,D])."""
    x = raw(qkv)
    xb = x.transpose(0, 1) if seq_major else x
    q, k, v = xb[:, :, :nh], xb[:, :, nh:nh + nkv], xb[:, :, nh + nkv:]
    if _bwd_backend[0] == "own" and x.is_contiguous() and fused_ok(q, k, v, None, 0.0, causal):
        sc = float(scale) if scale is not None else 1.0 / math.sqrt(x.shape[-1])
        return wrap(_FlashAttnPacked.apply(x, int(nh), int(nkv), sc, bool(causal), bool(seq_major)))
    out = attention(q, k, v, None, 0.0, causal, scale)
    return wrap(raw(out).transpose(0, 1).contiguous()) if seq_major else out


def fused_ok(q, k, v, mask, dropout_p, causal):
    if not (use_fused(q) and flag("FLAGS_b200_flash_attention", True)) or mask is not None or dropout_p != 0.0:
        return False
    if q.dtype not in (torch.float16, torch.bfloat16) or q.dim() != 4 or q.shape[-1] != 128:
        return False
    if causal and q.shape[1] != k.shape[1]:
        return False
    return bool(ext().attention_supported(q, k, v))


@recordable
def attention(q, k, v, mask=None, dropout_p=0.0, causal=False, scale=None):
    q, k, v, mask = raw(q), raw(k), raw(v), raw(mask)
    if fused_ok(q, k, v, mask, dropout_p, causal):
        sc = float(scale) if scale is not None else 1.0 / math.sqrt(q.shape[-1])
        return wrap(_FlashAttn.apply(q, k, v, sc, bool(causal)))
    if causal and mask is not None:
        sq, sk = q.shape[1], k.shape[1]
        cm = torch.ones(sq, sk, dtype=torch.bool, device=q.device).tril(sk - sq)
        mask = (mask & cm) if mask.dtype == torch.bool else mask.masked_fill(~cm, float("-inf"))
        causal = False
    return wrap(attention_ref(q, k, v, mask, dropout_p, causal, scale))
