"""Paged (block) KV-cache attention for serving. Parity: paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu
(python/paddle/incubate/nn/functional/block_multihead_attention.py)."""
from __future__ import annotations

import math

import torch

from ...tensor import Tensor


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


_PREFILL_BLOCK_SIZES = (16, 32, 64, 128, 256)


def _paged_kernels_ok(qkv, kc, d, block_size):
    from ...framework.flags import flag

    return (qkv.is_cuda and kc.is_cuda and d == 128 and qkv.dtype in (torch.float16, torch.bfloat16) and kc.dtype == qkv.dtype
            and int(block_size) in _PREFILL_BLOCK_SIZES and flag("FLAGS_use_fused_kernels", True))


def block_attention(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size):
    """qkv: [total_tokens, (H + 2*H_kv) * D] packed over the batch; caches [num_blocks, H_kv, block_size, D].

    A sequence prefills when seq_lens_encoder > 0 (a fresh prompt) or when it brings more than one token on top of seq_lens_decoder cached
    ones (a continuing chunk); it decodes when it brings exactly one token and seq_lens_encoder == 0.

    CUDA path (head_dim 128, fp16 / bf16, block_size 16 / 32 / 64 / 128 / 256): the new K / V rows of EVERY sequence are scattered into the
    paged caches with one indexed write (block and row computed on the device from the block table - no per-token Python loop); decode
    sequences attend to their cache through `decode_attention_paged` (csrc/decode_attention.cu: one table lookup per cached row, split-K
    over the positions); all prefill sequences run in ONE launch of `attention_fwd_paged` (csrc/attention_sm100.cu): causal wgmma flash
    attention of each sequence's new tokens over its whole cached prefix, K / V read in place through the block table, q read and the
    output written in place at the tokens' rows.  Other block sizes and devices take `_block_attention_ref`."""
    qkv, kc, vc = _raw(qkv), _raw(key_cache), _raw(value_cache)
    nkv, d = kc.shape[1], kc.shape[3]
    if not _paged_kernels_ok(qkv, kc, d, block_size):
        return _block_attention_ref(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size)
    from ..._build import ext

    dev = qkv.device
    nh = qkv.shape[1] // d - 2 * nkv
    enc = _raw(seq_lens_encoder).reshape(-1).to(dev, torch.int64)
    dec = _raw(seq_lens_decoder).reshape(-1).to(dev, torch.int64)
    now = _raw(seq_lens_this_time).reshape(-1).to(dev, torch.int64)
    cu = _raw(cu_seqlens_q).reshape(-1).to(dev, torch.int64)
    bt = _raw(block_tables).to(dev, torch.int32).contiguous()
    nseq = now.numel()
    total_tokens = qkv.shape[0]
    rows = qkv.reshape(total_tokens, nh + 2 * nkv, d)
    q, k, v = rows[:, :nh], rows[:, nh:nh + nkv], rows[:, nh + nkv:]
    # ---- scatter the new K / V rows into the paged caches (all sequences at once)
    tok = torch.arange(total_tokens, device=dev)
    seq_of = torch.bucketize(tok, cu[1:nseq + 1], right=True).clamp(max=nseq - 1)
    valid = tok < cu[nseq]
    past = torch.where(enc > 0, torch.zeros_like(dec), dec)                  # prefill starts at position 0, decode continues after the cache
    pos = past[seq_of] + (tok - cu[seq_of])
    blk = bt.long()[seq_of, (pos // block_size).clamp(max=bt.shape[1] - 1)]
    off = pos % block_size
    sel = valid.nonzero().reshape(-1)
    kc[blk[sel], :, off[sel]] = k[sel]
    vc[blk[sel], :, off[sel]] = v[sel]
    out = qkv.new_zeros((total_tokens, nh * d))
    scale = 1.0 / math.sqrt(d)
    is_dec = (now == 1) & (enc == 0)
    is_pre = (now > 0) & ~is_dec
    any_dec, any_pre = torch.stack([is_dec.any(), is_pre.any()]).tolist()
    # ---- decode sequences: one query token against the paged cache
    if any_dec:
        ids = is_dec.nonzero().reshape(-1)
        qd = q[cu[ids]].contiguous()                                        # [Bd, H, D]
        lens = (dec[ids] + 1).to(torch.int32).contiguous()
        od = ext().decode_attention_paged(qd, kc, vc, lens, bt[ids].contiguous(), scale)
        out[cu[ids]] = od.reshape(ids.numel(), nh * d)
    # ---- prefill sequences (fresh prompts and continuing chunks): new tokens over their whole cached prefix, one launch for all
    if any_pre:
        i32 = lambda t: t.to(torch.int32).contiguous()                      # noqa: E731
        ext().attention_fwd_paged(q, kc, vc, bt, i32(cu[:nseq]), i32(torch.where(is_pre, now, 0)), i32(past), scale, out)
    return out.as_subclass(Tensor), qkv.as_subclass(Tensor), kc.as_subclass(Tensor), vc.as_subclass(Tensor)


def _block_attention_ref(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size):
    """qkv: [total_tokens, (H + 2*H_kv) * D] packed over the batch; caches [num_blocks, H_kv, block_size, D]."""
    qkv, kc, vc = _raw(qkv), _raw(key_cache), _raw(value_cache)
    nkv, d = kc.shape[1], kc.shape[3]
    nh = qkv.shape[1] // d - 2 * nkv
    enc, dec, now = _raw(seq_lens_encoder).reshape(-1).tolist(), _raw(seq_lens_decoder).reshape(-1).tolist(), _raw(seq_lens_this_time).reshape(-1).tolist()
    cu = _raw(cu_seqlens_q).reshape(-1).tolist()
    bt = _raw(block_tables)
    out = qkv.new_zeros((qkv.shape[0], nh * d))
    for b in range(len(now)):
        n = now[b]
        if n == 0:
            continue
        rows = qkv[cu[b]:cu[b] + n].reshape(n, nh + 2 * nkv, d)
        q, k, v = rows[:, :nh], rows[:, nh:nh + nkv], rows[:, nh + nkv:]
        past = dec[b] if enc[b] == 0 else 0
        for t in range(n):  # append new K/V into the paged cache
            pos = past + t
            blk, off = int(bt[b, pos // block_size]), pos % block_size
            kc[blk, :, off] = k[t]
            vc[blk, :, off] = v[t]
        total = past + n
        nblk = (total + block_size - 1) // block_size
        blks = bt[b, :nblk].long()
        K = kc[blks].permute(1, 0, 2, 3).reshape(nkv, nblk * block_size, d)[:, :total]
        V = vc[blks].permute(1, 0, 2, 3).reshape(nkv, nblk * block_size, d)[:, :total]
        rep = nh // nkv
        K, V = K.repeat_interleave(rep, 0), V.repeat_interleave(rep, 0)
        s = torch.einsum("nhd,hsd->hns", q.float(), K.float()) / math.sqrt(d)
        qpos = torch.arange(past, total, device=qkv.device)[None, :, None]
        kpos = torch.arange(total, device=qkv.device)[None, None, :]
        s = s.masked_fill(kpos > qpos, float("-inf"))
        o = torch.einsum("hns,hsd->nhd", torch.softmax(s, -1), V.float())
        out[cu[b]:cu[b] + n] = o.reshape(n, nh * d).to(out.dtype)
    return out.as_subclass(Tensor), qkv.as_subclass(Tensor), kc.as_subclass(Tensor), vc.as_subclass(Tensor)
