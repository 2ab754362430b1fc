"""Attention functionals. Parity: python/paddle/nn/functional/flash_attention.py, sparse_attention.py.

Layout is paddle's: q/k/v are [batch, seqlen, num_heads, head_dim].
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from ...ops._helpers import T, raw, wrap


def scaled_dot_product_attention(query, key, value, attn_mask=None, dropout_p=0.0, is_causal=False, training=True,
                                 backend=None, scale=None, enable_gqa=True, name=None):
    from ...kernels import attention as K

    return K.attention(T(query), T(key), T(value), attn_mask, dropout_p if training else 0.0, is_causal, scale)


def flash_attention(query, key, value, dropout=0.0, causal=False, return_softmax=False, fixed_seed_offset=None,
                    rng_name="", training=True, name=None):
    from ...kernels import attention as K

    out = K.attention(T(query), T(key), T(value), None, dropout if training else 0.0, causal, None, seed_offset=fixed_seed_offset)
    return out, None


def flash_attn_qkvpacked(qkv, dropout=0.0, causal=False, return_softmax=False, fixed_seed_offset=None, rng_name="",
                         training=True, name=None):
    qkv = T(qkv)  # [B, S, G+2, Hk, D]
    g = qkv.size(2) - 2
    b, s, _, hk, d = qkv.size()
    q = qkv[:, :, :g].reshape(b, s, g * hk, d)
    return flash_attention(q, qkv[:, :, g], qkv[:, :, g + 1], dropout, causal, return_softmax, fixed_seed_offset=fixed_seed_offset, training=training)


def flash_attn_unpadded(query, key, value, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale,
                        dropout=0.0, causal=False, return_softmax=False, fixed_seed_offset=None, rng_name="",
                        training=True, name=None):
    """Varlen attention over packed [total_tokens, H, D]. Parity: flash_attention.py:flash_attn_unpadded."""
    from ...kernels import attention as K

    q, k, v = T(query), T(key), T(value)
    p = dropout if training else 0.0
    if q.is_cuda and q.dim() == 3:
        # packed batch as ONE sequence under a document mask: no host read of cu_seqlens, no per-sequence launches.
        # (causal: the diagonal of every sequence is the global diagonal when q and k are packed alike - self attention; otherwise the
        # mask carries each sequence's own bottom-right aligned causal limit and the kernels run without theirs)
        same = cu_seqlens_q is cu_seqlens_k or (raw(cu_seqlens_q).shape == raw(cu_seqlens_k).shape and q.size(0) == k.size(0))
        cm = K.colmask_from_cu_seqlens(cu_seqlens_q, cu_seqlens_k, k.size(0), causal=causal and not same)
        out = K.attention_colmask(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), cm, causal and same, scale, p, fixed_seed_offset)
        if out is not None:
            return out.squeeze(0), None
    cq, ck = raw(cu_seqlens_q).tolist(), raw(cu_seqlens_k).tolist()
    outs = []
    for i in range(len(cq) - 1):
        qi, ki, vi = q[cq[i]:cq[i + 1]], k[ck[i]:ck[i + 1]], v[ck[i]:ck[i + 1]]
        outs.append(K.attention(qi.unsqueeze(0), ki.unsqueeze(0), vi.unsqueeze(0), None, p, causal, scale).squeeze(0))
    return torch.cat(outs, 0), None


def flash_attn_varlen_qkvpacked(qkv, cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale, dropout=0.0,
                                causal=False, return_softmax=False, fixed_seed_offset=None, rng_name="", varlen_padded=True,
                                training=True, name=None):
    qkv = T(qkv)
    g = qkv.size(1) - 2
    t, _, hk, d = qkv.size()
    q = qkv[:, :g].reshape(t, g * hk, d)
    return flash_attn_unpadded(q, qkv[:, g], qkv[:, g + 1], cu_seqlens_q, cu_seqlens_k, max_seqlen_q, max_seqlen_k, scale, dropout, causal,
                               fixed_seed_offset=fixed_seed_offset, training=training)


def flashmask_attention(query, key, value, startend_row_indices=None, dropout=0.0, causal=False, window_size=None,
                        return_softmax_lse=False, return_seed_offset=False, fixed_seed_offset=None, rng_name="",
                        training=True, name=None):
    """Column-wise sparse mask attention. Parity: flash_attention.py:flashmask_attention.

    startend_row_indices: [B, Hm, S_k, {1,2,4}] int32; for key column j, rows in [LTS, LTE) (lower triangle) and
    [UTS, UTE) (upper) are masked.  Dropout in training runs on the own kernels; fixed_seed_offset (int64 [2]) fixes its mask, and
    return_seed_offset=True returns [out, seed_offset], the pair that reproduces it.
    """
    from ...kernels import attention as K

    q, k, v = T(query), T(key), T(value)
    sq, sk = q.size(1), k.size(1)
    mask = None
    p = dropout if training else 0.0
    if q.is_cuda and (startend_row_indices is not None or window_size is not None):
        if startend_row_indices is not None:
            cm = K.colmask_from_startend(startend_row_indices, causal, sq)
        else:
            w = (window_size, window_size) if isinstance(window_size, int) else tuple(window_size)
            cm = K.colmask_from_window(sq, sk, int(w[0]), int(w[1]), causal, q.device)
        if cm.shape[0] == 1 and q.size(0) > 1:
            cm = cm.expand(q.size(0), -1, -1, -1).contiguous()
        res = K.attention_colmask(q, k, v, cm, causal, None, p, fixed_seed_offset, return_seed_offset=True)
        if res is not None:
            return [res[0], res[1]] if return_seed_offset else res[0]
    elif startend_row_indices is None and window_size is None:
        res = K.attention(q, k, v, None, p, causal, None, seed_offset=fixed_seed_offset, return_seed_offset=return_seed_offset and K.fused_ok(
            raw(q), raw(k), raw(v), None, p, causal))
        if return_seed_offset:
            return [res[0], res[1]] if isinstance(res, tuple) else [res, None]
        return res
    if startend_row_indices is not None:
        idx = raw(startend_row_indices).long()
        rows = torch.arange(sq, device=q.device).reshape(1, 1, sq, 1)
        n = idx.size(-1)
        lts = idx[..., 0].unsqueeze(2)
        if causal:
            lte = idx[..., 1].unsqueeze(2) if n == 2 else None
            masked = (rows >= lts) & ((rows < lte) if lte is not None else True)
        else:
            if n == 2:
                ute = idx[..., 1].unsqueeze(2)
                masked = (rows >= lts) | (rows < ute)
            elif n == 4:
                lte, uts, ute = idx[..., 1].unsqueeze(2), idx[..., 2].unsqueeze(2), idx[..., 3].unsqueeze(2)
                masked = ((rows >= lts) & (rows < lte)) | ((rows >= uts) & (rows < ute))
            else:
                masked = rows >= lts
        mask = ~masked
        if causal:
            mask = mask & torch.ones(sq, sk, dtype=torch.bool, device=q.device).tril(sk - sq)
    elif window_size is not None:
        w = (window_size, window_size) if isinstance(window_size, int) else tuple(window_size)
        i = torch.arange(sq, device=q.device).unsqueeze(1)
        j = torch.arange(sk, device=q.device).unsqueeze(0)
        mask = (j >= i - w[0]) & ((j <= i + w[1]) if not causal else (j <= i))
        mask = mask.reshape(1, 1, sq, sk)
    out = K.attention(q, k, v, mask, p, causal and mask is None, None)
    return [out, None] if return_seed_offset else out


def calc_reduced_attention_scores(query, key, softmax_lse, name=None):
    q, k = T(query), T(key)
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) / math.sqrt(q.size(-1))
    p = torch.exp(s - raw(softmax_lse).unsqueeze(-1))
    return p.sum(2, keepdim=True)


def sparse_attention(query, key, value, sparse_csr_offset, sparse_csr_columns, key_padding_mask=None, attn_mask=None, name=None):
    """Block-CSR sparse attention ([B,H,S,D] layout). Parity: nn/functional/sparse_attention.py."""
    q, k, v = T(query), T(key), T(value)
    b, h, s, d = q.size()
    off, col = raw(sparse_csr_offset).long(), raw(sparse_csr_columns).long()
    mask = torch.zeros(b, h, s, s, dtype=torch.bool, device=q.device)
    for bi in range(b):
        for hi in range(h):
            o, c = off[bi, hi], col[bi, hi]
            rows = torch.repeat_interleave(torch.arange(s, device=q.device), o[1:] - o[:-1])
            mask[bi, hi, rows, c[: rows.numel()]] = True
    scores = (q @ k.transpose(-1, -2)) / math.sqrt(d)
    scores = scores.masked_fill(~mask, float("-inf"))
    if key_padding_mask is not None:
        scores = scores + T(key_padding_mask).reshape(b, 1, 1, s)
    if attn_mask is not None:
        scores = scores + T(attn_mask).reshape(1, 1, s, s)
    return torch.softmax(scores, -1) @ v


def sdp_kernel(*a, **k):
    import contextlib

    return contextlib.nullcontext()


__all__ = ["scaled_dot_product_attention", "flash_attention", "flash_attn_qkvpacked", "flash_attn_unpadded",
           "flash_attn_varlen_qkvpacked", "flashmask_attention", "calc_reduced_attention_scores", "sparse_attention", "sdp_kernel"]
