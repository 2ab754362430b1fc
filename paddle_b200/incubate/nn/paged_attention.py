"""Paged (block) KV-cache attention for serving. Parity: paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu
(python/paddle/incubate/nn/functional/block_multihead_attention.py).

Quantized caches: int8 or float8_e4m3fn caches with static per-KV-head scales (fp32 [H_kv], one quant / dequant pair each for K and V).
A new row is stored as y = (quant_max_bound * quant_scale[h]) * x in fp32; int8 rounds it (quant_round_type 0: half to even, 1: half
away from zero) and then clamps it to [quant_min_bound, quant_max_bound]; fp8 clamps it and then rounds to nearest even.  A cached value
q is read back as q * dequant_scale[h].  The reference path and the CUDA kernels apply these rules bit for bit alike."""
from __future__ import annotations

import math
from typing import NamedTuple

import torch

from ...tensor import Tensor


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


_PREFILL_BLOCK_SIZES = (16, 32, 64, 128, 256)
# Longest continuing chunk (seq_lens_encoder == 0) that block_attention sends to `decode_attention_paged_multi` rather than
# `attention_fwd_paged`; also capped so that now * (H / H_kv) <= 64.  Set from scripts/bench_spec_verify.py (DESIGN.md section 4).
VERIFY_MAX = 16
_KV8_DTYPES = (torch.int8, torch.float8_e4m3fn)
_KV8_LIMITS = {torch.int8: (-128.0, 127.0), torch.float8_e4m3fn: (-448.0, 448.0)}


class KVQuant(NamedTuple):
    """Validated static cache quantization: fp32 [H_kv] scales on the caches' device, and the rounding rule."""
    k_quant: torch.Tensor
    v_quant: torch.Tensor
    k_dequant: torch.Tensor
    v_dequant: torch.Tensor
    round_type: int
    max_bound: float
    min_bound: float


def kv_quant_params(key_cache, value_cache, cache_k_quant_scales=None, cache_v_quant_scales=None, cache_k_dequant_scales=None,
                    cache_v_dequant_scales=None, use_dynamic_cachekv_quant=False, quant_round_type=1, quant_max_bound=127.0, quant_min_bound=-127.0):
    """None for 16-bit caches, a KVQuant for int8 / float8_e4m3fn caches.  Raises on inputs that would otherwise be silently wrong."""
    kc, vc = _raw(key_cache), _raw(value_cache)
    scales = [_raw(t) for t in (cache_k_quant_scales, cache_v_quant_scales, cache_k_dequant_scales, cache_v_dequant_scales)]
    if use_dynamic_cachekv_quant:
        raise NotImplementedError("block_multihead_attention: dynamic (per batch and head) cache-KV quantization is not implemented; "
                                  "use static per-KV-head scales")
    if kc.dtype != vc.dtype and (kc.dtype in _KV8_DTYPES or vc.dtype in _KV8_DTYPES):
        raise ValueError(f"block_multihead_attention: key and value caches differ in dtype ({kc.dtype} and {vc.dtype})")
    if kc.dtype not in _KV8_DTYPES:
        if any(t is not None for t in scales):
            raise ValueError(f"block_multihead_attention: cache quant / dequant scales were given with a {kc.dtype} cache; "
                             "they need an int8 or float8_e4m3fn cache")
        return None
    if any(t is None for t in scales):
        raise ValueError(f"block_multihead_attention: a {kc.dtype} cache needs cache_k_quant_scales, cache_v_quant_scales, "
                         "cache_k_dequant_scales and cache_v_dequant_scales")
    nkv = kc.shape[1]
    for t in scales:
        if tuple(t.shape) != (nkv,):
            raise ValueError(f"block_multihead_attention: static cache scales must have shape [H_kv] = [{nkv}], got {list(t.shape)}")
    if int(quant_round_type) not in (0, 1):
        raise ValueError(f"block_multihead_attention: quant_round_type must be 0 or 1, got {quant_round_type}")
    lo, hi = _KV8_LIMITS[kc.dtype]
    if not (lo <= float(quant_min_bound) <= float(quant_max_bound) <= hi):
        raise ValueError(f"block_multihead_attention: quant bounds [{quant_min_bound}, {quant_max_bound}] must lie within [{lo}, {hi}] "
                         f"for a {kc.dtype} cache")
    f32 = [t.to(kc.device, torch.float32).contiguous() for t in scales]
    return KVQuant(*f32, int(quant_round_type), float(quant_max_bound), float(quant_min_bound))


def _round_half_away(y):
    """roundf: ties away from zero.  y - trunc(y) is exact in fp32, so 0.49999997 stays below one half (floor(|y| + 0.5) rounds it up)."""
    t = torch.trunc(y)
    return t + torch.sign(y) * ((y - t).abs() >= 0.5).to(y.dtype)


def quantize_kv(x, quant_scale, quant, dtype):
    """x [..., H_kv, D] -> `dtype` (int8 / float8_e4m3fn) under the static rules of this module (fp32 arithmetic throughout)."""
    a = torch.tensor(quant.max_bound, dtype=torch.float32, device=x.device) * quant_scale.to(x.device, torch.float32)
    y = a[:, None] * x.float()
    if dtype == torch.int8:
        y = torch.round(y) if quant.round_type == 0 else _round_half_away(y)
        return y.clamp(quant.min_bound, quant.max_bound).to(torch.int8)
    return y.clamp(quant.min_bound, quant.max_bound).to(dtype)


def dequantize_kv(q, dequant_scale):
    """q [H_kv, S, D] 8-bit -> fp32 q * dequant_scale[h]."""
    return q.float() * dequant_scale.to(q.device, torch.float32)[:, None, None]


def _paged_kernels_ok(qkv, kc, d, block_size, quant=None):
    from ...framework.flags import flag

    cache_ok = kc.dtype == qkv.dtype or (quant is not None and kc.dtype in _KV8_DTYPES)
    return (qkv.is_cuda and kc.is_cuda and d == 128 and qkv.dtype in (torch.float16, torch.bfloat16) and cache_ok
            and int(block_size) in _PREFILL_BLOCK_SIZES and flag("FLAGS_use_fused_kernels", True))


def block_attention(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size,
                    cache_k_quant_scales=None, cache_v_quant_scales=None, cache_k_dequant_scales=None, cache_v_dequant_scales=None,
                    use_dynamic_cachekv_quant=False, quant_round_type=1, quant_max_bound=127.0, quant_min_bound=-127.0):
    """qkv: [total_tokens, (H + 2*H_kv) * D] packed over the batch; caches [num_blocks, H_kv, block_size, D].

    A sequence prefills when seq_lens_encoder > 0 (a fresh prompt) or when it brings more than one token on top of seq_lens_decoder cached
    ones (a continuing chunk); it decodes when it brings exactly one token and seq_lens_encoder == 0.  A continuing chunk of 2 ..
    VERIFY_MAX tokens with now * (H / H_kv) <= 64 - the verify rows of speculative decoding - is a short chunk.

    CUDA path (head_dim 128, fp16 / bf16, block_size 16 / 32 / 64 / 128 / 256): the new K / V rows of EVERY sequence are scattered into the
    paged caches with one indexed write (block and row computed on the device from the block table - no per-token Python loop); decode
    sequences attend to their cache through `decode_attention_paged` (csrc/decode_attention.cu: one table lookup per cached row, split-K
    over the positions); all prefill sequences run in ONE launch of `attention_fwd_paged` (csrc/attention_sm100.cu): causal wgmma flash
    attention of each sequence's new tokens over its whole cached prefix, K / V read in place through the block table, q read and the
    output written in place at the tokens' rows; all short chunks run in ONE launch of `decode_attention_paged_multi`
    (csrc/decode_attention.cu: split-K over the cached positions, every query row of a KV head in one tensor-core tile, q and the output in
    place as for prefill).  The three row kinds are told apart with one host read.  Other block sizes and devices take
    `_block_attention_ref`.

    int8 / float8_e4m3fn caches (static scales, see the module docstring): the new rows are quantized into the caches by one launch of
    `paged_kv_cache_write` (csrc/kv_cache_quant.cu), and the attention kernels read the 8-bit rows and dequantize them on the fly."""
    qkv, kc, vc = _raw(qkv), _raw(key_cache), _raw(value_cache)
    nkv, d = kc.shape[1], kc.shape[3]
    quant = kv_quant_params(kc, vc, cache_k_quant_scales, cache_v_quant_scales, cache_k_dequant_scales, cache_v_dequant_scales,
                            use_dynamic_cachekv_quant, quant_round_type, quant_max_bound, quant_min_bound)
    if not _paged_kernels_ok(qkv, kc, d, block_size, quant):
        return _block_attention_ref(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables,
                                    block_size, quant=quant)
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
    past = torch.where(enc > 0, torch.zeros_like(dec), dec)                  # prefill starts at position 0, decode continues after the cache
    i32 = lambda t: t.to(torch.int32).contiguous()                          # noqa: E731
    if quant is None:
        # ---- scatter the new K / V rows into the paged caches (all sequences at once)
        tok = torch.arange(total_tokens, device=dev)
        seq_of = torch.bucketize(tok, cu[1:nseq + 1], right=True).clamp(max=nseq - 1)
        valid = tok < cu[nseq]
        pos = past[seq_of] + (tok - cu[seq_of])
        blk = bt.long()[seq_of, (pos // block_size).clamp(max=bt.shape[1] - 1)]
        off = pos % block_size
        sel = valid.nonzero().reshape(-1)
        kc[blk[sel], :, off[sel]] = k[sel]
        vc[blk[sel], :, off[sel]] = v[sel]
        dq = {}
    else:
        # ---- quantize the new K / V rows into the 8-bit caches: one launch, rows read in place from qkv
        ext().paged_kv_cache_write(qkv.reshape(total_tokens, -1), kc, vc, i32(cu[:nseq + 1]), i32(enc), i32(dec), bt, quant.k_quant, quant.v_quant,
                                   quant.round_type, quant.max_bound, quant.min_bound)
        dq = {"k_dequant_scales": quant.k_dequant, "v_dequant_scales": quant.v_dequant}
    out = qkv.new_zeros((total_tokens, nh * d))
    scale = 1.0 / math.sqrt(d)
    is_dec = (now == 1) & (enc == 0)
    is_ver = (enc == 0) & (now >= 2) & (now <= min(VERIFY_MAX, 64 // (nh // nkv)))
    is_pre = (now > 0) & ~is_dec & ~is_ver
    any_dec, any_ver, any_pre = torch.stack([is_dec.any(), is_ver.any(), is_pre.any()]).tolist()
    # ---- decode sequences: one query token against the paged cache
    if any_dec:
        ids = is_dec.nonzero().reshape(-1)
        qd = q[cu[ids]].contiguous()                                        # [Bd, H, D]
        lens = (dec[ids] + 1).to(torch.int32).contiguous()
        od = ext().decode_attention_paged(qd, kc, vc, lens, bt[ids].contiguous(), scale, **dq)
        out[cu[ids]] = od.reshape(ids.numel(), nh * d)
    # ---- short chunks (verify rows): a few new tokens over a long cached prefix, one launch for all
    if any_ver:
        ext().decode_attention_paged_multi(q, kc, vc, bt, i32(cu[:nseq]), i32(torch.where(is_ver, now, 0)), i32(past), scale, out, **dq)
    # ---- prefill sequences (fresh prompts and longer continuing chunks): new tokens over their whole cached prefix, one launch for all
    if any_pre:
        ext().attention_fwd_paged(q, kc, vc, bt, i32(cu[:nseq]), i32(torch.where(is_pre, now, 0)), i32(past), scale, out, **dq)
    return out.as_subclass(Tensor), qkv.as_subclass(Tensor), kc.as_subclass(Tensor), vc.as_subclass(Tensor)


def _block_attention_ref(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size,
                         cache_k_quant_scales=None, cache_v_quant_scales=None, cache_k_dequant_scales=None, cache_v_dequant_scales=None,
                         use_dynamic_cachekv_quant=False, quant_round_type=1, quant_max_bound=127.0, quant_min_bound=-127.0, quant=None):
    """qkv: [total_tokens, (H + 2*H_kv) * D] packed over the batch; caches [num_blocks, H_kv, block_size, D].  `quant`: an already
    validated KVQuant (otherwise it is built from the scale / round / bound arguments)."""
    qkv, kc, vc = _raw(qkv), _raw(key_cache), _raw(value_cache)
    if quant is None:
        quant = kv_quant_params(kc, vc, cache_k_quant_scales, cache_v_quant_scales, cache_k_dequant_scales, cache_v_dequant_scales,
                                use_dynamic_cachekv_quant, quant_round_type, quant_max_bound, quant_min_bound)
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
            if quant is None:
                kc[blk, :, off] = k[t]
                vc[blk, :, off] = v[t]
            else:
                kc[blk, :, off] = quantize_kv(k[t], quant.k_quant, quant, kc.dtype)
                vc[blk, :, off] = quantize_kv(v[t], quant.v_quant, quant, vc.dtype)
        total = past + n
        nblk = (total + block_size - 1) // block_size
        blks = bt[b, :nblk].long()
        K = kc[blks].permute(1, 0, 2, 3).reshape(nkv, nblk * block_size, d)[:, :total]
        V = vc[blks].permute(1, 0, 2, 3).reshape(nkv, nblk * block_size, d)[:, :total]
        if quant is not None:
            K, V = dequantize_kv(K, quant.k_dequant), dequantize_kv(V, quant.v_dequant)
        rep = nh // nkv
        K, V = K.repeat_interleave(rep, 0), V.repeat_interleave(rep, 0)
        s = torch.einsum("nhd,hsd->hns", q.float(), K.float()) / math.sqrt(d)
        qpos = torch.arange(past, total, device=qkv.device)[None, :, None]
        kpos = torch.arange(total, device=qkv.device)[None, None, :]
        s = s.masked_fill(kpos > qpos, float("-inf"))
        o = torch.einsum("hns,hsd->nhd", torch.softmax(s, -1), V.float())
        out[cu[b]:cu[b] + n] = o.reshape(n, nh * d).to(out.dtype)
    return out.as_subclass(Tensor), qkv.as_subclass(Tensor), kc.as_subclass(Tensor), vc.as_subclass(Tensor)
