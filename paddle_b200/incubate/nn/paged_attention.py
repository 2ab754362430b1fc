"""Paged (block) KV-cache attention for serving. Parity: paddle/phi/kernels/fusion/gpu/block_multi_head_attention_kernel.cu
(python/paddle/incubate/nn/functional/block_multihead_attention.py).

CUDA kernels serve head_dim 128 and, over fp16 / bf16 caches, head_dim 64 (the 1B-class models used as speculative drafts); see
block_attention for what stays on the reference path.

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
# Decode rows that share a cached prefix run on `decode_attention_paged_shared` only in groups of at least SHARED_PREFIX_MIN_GROUP
# sequences sharing at least SHARED_PREFIX_MIN_TOKENS prefix tokens; smaller groups stay on `decode_attention_paged`.  Set from
# scripts/bench_prefix_caching.py (DESIGN.md section 4).
SHARED_PREFIX_MIN_GROUP = 4
SHARED_PREFIX_MIN_TOKENS = 4096
# ... or of at least SHARED_PREFIX_LARGE_GROUP sequences sharing at least SHARED_PREFIX_LARGE_GROUP_MIN_TOKENS.
SHARED_PREFIX_LARGE_GROUP = 16
SHARED_PREFIX_LARGE_GROUP_MIN_TOKENS = 512
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


class QKVPrologue(NamedTuple):
    """Validated qkv prologue / output epilogue of block_multihead_attention (see block_attention), on qkv's device.  dtype: the compute type
    T.  qkv_out_scale: fp32 [W] (int32 qkv only); qkv_bias: T [W]; rope_cos / rope_sin: fp32 [S_rope, R] with neox; out_dtype: int8 /
    float8_e4m3fn when out_scale > 0, else None; out_shift / out_smooth: T [H * D]."""
    dtype: torch.dtype
    qkv_out_scale: torch.Tensor | None
    qkv_bias: torch.Tensor | None
    rope_cos: torch.Tensor | None
    rope_sin: torch.Tensor | None
    neox: bool
    out_scale: float
    out_dtype: torch.dtype | None
    out_shift: torch.Tensor | None
    out_smooth: torch.Tensor | None
    round_type: int
    max_bound: float
    min_bound: float

    @property
    def has_prologue(self):
        return self.qkv_out_scale is not None or self.qkv_bias is not None or self.rope_cos is not None


_COMPUTE_DTYPES = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}
_OUT_DTYPES = {127.0: torch.int8, 448.0: torch.float8_e4m3fn}


def qkv_prologue_params(qkv, num_heads, num_kv_heads, head_dim, qkv_out_scale=None, qkv_bias=None, rope_emb=None, use_neox_style=False,
                        out_shift=None, out_smooth=None, out_scale=-1, compute_dtype="default", quant_round_type=1, quant_max_bound=127.0,
                        quant_min_bound=-127.0):
    """None when block_attention's qkv prologue and output epilogue have nothing to do (no int32 qkv, qkv_bias, rope_emb, and out_scale
    <= 0), else a QKVPrologue.  Raises ValueError on inputs the op would otherwise get silently wrong."""
    qkv = _raw(qkv)
    qkv_out_scale, qkv_bias, rope_emb, out_shift, out_smooth = (_raw(t) for t in (qkv_out_scale, qkv_bias, rope_emb, out_shift, out_smooth))
    dev, w = qkv.device, qkv.shape[1]
    if compute_dtype != "default" and compute_dtype not in _COMPUTE_DTYPES:
        raise ValueError(f"block_multihead_attention: compute_dtype must be 'default', 'bf16', 'fp16' or 'fp32', got {compute_dtype!r}")
    if qkv.dtype == torch.int32:
        if compute_dtype == "default":
            raise ValueError("block_multihead_attention: int32 qkv needs compute_dtype 'bf16', 'fp16' or 'fp32'")
        if qkv_out_scale is None:
            raise ValueError("block_multihead_attention: int32 qkv needs qkv_out_scale (fp32 [W]) to dequantize it")
        dtype = _COMPUTE_DTYPES[compute_dtype]
        if qkv_out_scale.numel() != w:
            raise ValueError(f"block_multihead_attention: qkv_out_scale must have W = {w} elements, got {list(qkv_out_scale.shape)}")
        qkv_out_scale = qkv_out_scale.reshape(w).to(dev, torch.float32).contiguous()
    else:
        if qkv_out_scale is not None:
            raise ValueError(f"block_multihead_attention: qkv_out_scale dequantizes int32 qkv; qkv is {qkv.dtype}")
        if compute_dtype != "default" and _COMPUTE_DTYPES[compute_dtype] != qkv.dtype:
            raise ValueError(f"block_multihead_attention: compute_dtype {compute_dtype!r} does not match the {qkv.dtype} qkv")
        dtype = qkv.dtype
    if qkv_bias is not None:
        if qkv_bias.numel() != w:
            raise ValueError(f"block_multihead_attention: qkv_bias must have W = {w} elements, got {list(qkv_bias.shape)}")
        qkv_bias = qkv_bias.reshape(w).to(dev, dtype).contiguous()
    cos = sin = None
    if rope_emb is not None:
        r = head_dim if use_neox_style else head_dim // 2
        if rope_emb.dim() != 5 or rope_emb.shape[0] != 2 or rope_emb.shape[3] != 1:
            raise ValueError(f"block_multihead_attention: rope_emb must be [2, 1, S, 1, {r}] (cos, sin), got {list(rope_emb.shape)}")
        if rope_emb.shape[1] != 1:
            raise ValueError(f"block_multihead_attention: rope_emb must have batch dimension 1 (one table for every sequence), got "
                             f"{rope_emb.shape[1]}")
        if rope_emb.shape[4] != r:
            raise ValueError(f"block_multihead_attention: rope_emb's last dimension must be {r} (head_dim{'' if use_neox_style else ' / 2'} "
                             f"with use_neox_style={bool(use_neox_style)}), got {rope_emb.shape[4]}")
        t = rope_emb.to(dev, torch.float32)
        cos, sin = t[0].reshape(-1, r).contiguous(), t[1].reshape(-1, r).contiguous()
    out_dtype = None
    if float(out_scale) > 0:
        out_dtype = _OUT_DTYPES.get(float(quant_max_bound))
        if out_dtype is None:
            raise ValueError(f"block_multihead_attention: out_scale > 0 needs quant_max_bound 127 (int8 output) or 448 (float8_e4m3fn output), "
                             f"got {quant_max_bound}")
        lo, hi = _KV8_LIMITS[out_dtype]
        if not (lo <= float(quant_min_bound) <= float(quant_max_bound)):
            raise ValueError(f"block_multihead_attention: quant_min_bound {quant_min_bound} must lie within [{lo}, {quant_max_bound}]")
        if int(quant_round_type) not in (0, 1):
            raise ValueError(f"block_multihead_attention: quant_round_type must be 0 or 1, got {quant_round_type}")
        if (out_shift is None) != (out_smooth is None):
            raise ValueError("block_multihead_attention: out_shift and out_smooth go together")
        if out_shift is not None:
            if out_dtype != torch.int8:
                raise ValueError("block_multihead_attention: out_shift / out_smooth apply to int8 output only (quant_max_bound 127)")
            hd = num_heads * head_dim
            if out_shift.numel() != hd or out_smooth.numel() != hd:
                raise ValueError(f"block_multihead_attention: out_shift / out_smooth must have H * D = {hd} elements")
            out_shift, out_smooth = out_shift.reshape(hd).to(dev, dtype).contiguous(), out_smooth.reshape(hd).to(dev, dtype).contiguous()
    else:
        out_shift = out_smooth = None                                          # as in the reference: not applied without out_scale
    if qkv.dtype != torch.int32 and qkv_bias is None and cos is None and out_dtype is None:
        return None
    return QKVPrologue(dtype, qkv_out_scale, qkv_bias, cos, sin, bool(use_neox_style), float(out_scale), out_dtype, out_shift, out_smooth,
                       int(quant_round_type), float(quant_max_bound), float(quant_min_bound))


def _prologue_ref(x, pro, pos, nh, nkv, d):
    """The qkv prologue op by op in torch: x [n, W] packed rows (int32 or T), pos [n] their positions -> processed rows [n, W] of T."""
    if x.dtype == torch.int32:
        x = (x.float() * pro.qkv_out_scale).to(pro.dtype)
    if pro.qkv_bias is not None:
        x = x + pro.qkv_bias
    if pro.rope_cos is None:
        return x
    n = x.shape[0]
    rows = x.reshape(n, nh + 2 * nkv, d)
    qk = rows[:, :nh + nkv].float()
    c, s = pro.rope_cos[pos][:, None, :d // 2], pro.rope_sin[pos][:, None, :d // 2]
    if pro.neox:
        l, r = qk[..., :d // 2], qk[..., d // 2:]
    else:
        l, r = qk[..., 0::2], qk[..., 1::2]
    nl, nr = l * c - r * s, r * c + l * s
    qk = torch.cat([nl, nr], -1) if pro.neox else torch.stack([nl, nr], -1).flatten(-2)
    return torch.cat([qk.to(pro.dtype), rows[:, nh + nkv:]], 1).reshape(n, -1)


def _out_quant_ref(o, pro):
    """The out_scale epilogue op by op: o [T, H * D] of T -> int8 / float8_e4m3fn."""
    if pro.out_shift is not None:
        o = (o + pro.out_shift) * pro.out_smooth
    a = torch.tensor(pro.max_bound, dtype=torch.float32, device=o.device) * torch.tensor(pro.out_scale, dtype=torch.float32, device=o.device)
    y = a * o.float()
    if pro.out_dtype == torch.int8:
        y = torch.round(y) if pro.round_type == 0 else _round_half_away(y)
        return y.clamp(pro.min_bound, pro.max_bound).to(torch.int8)
    return y.clamp(pro.min_bound, pro.max_bound).to(pro.out_dtype)


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


def shared_prefix_pays(group_size, prefix_len, heads_per_kv):
    """Whether a group of `group_size` decode rows sharing `prefix_len` cached tokens is worth `decode_attention_paged_shared`.  On an H100
    (DESIGN.md section 4) it lost to `decode_attention_paged` in groups of 2 at every prefix with 32 / 32 heads and an int8 cache, and in
    groups of 2 and 4 at 512 - 1024 prefix tokens; it won in every measured group of 4 from 4096 tokens and of 16 from 512.  heads_per_kv
    (H / H_kv) is not used: those break-even points held for 32 / 8 and 32 / 32 heads alike."""
    return ((group_size >= SHARED_PREFIX_MIN_GROUP and prefix_len >= SHARED_PREFIX_MIN_TOKENS)
            or (group_size >= SHARED_PREFIX_LARGE_GROUP and prefix_len >= SHARED_PREFIX_LARGE_GROUP_MIN_TOKENS))


def _shared_prefix_groups(shared_prefix, nseq, block_size):
    """Validates the host-visible part of block_attention's shared_prefix = (cu_groups [G+1], group_seqs [n], prefix_len [G]) (host
    lists or CPU integer tensors) and returns them as int lists.  Raises ValueError."""
    def as_list(v, name):
        if isinstance(v, torch.Tensor):
            v = _raw(v)
            if v.device.type != "cpu" or v.dtype not in (torch.int32, torch.int64) or v.dim() != 1:
                raise ValueError(f"shared_prefix: {name} must be a host list or a 1-D CPU integer tensor")
            return v.tolist()
        return [int(x) for x in v]

    try:
        cu, seqs, plen = shared_prefix
    except (TypeError, ValueError):
        raise ValueError("shared_prefix must be (cu_groups, group_seqs, prefix_len)") from None
    cu, seqs, plen = as_list(cu, "cu_groups"), as_list(seqs, "group_seqs"), as_list(plen, "prefix_len")
    if len(cu) != len(plen) + 1 or not cu or cu[0] != 0 or cu[-1] != len(seqs) or any(b <= a for a, b in zip(cu, cu[1:])):
        raise ValueError(f"shared_prefix: cu_groups must rise strictly from 0 to len(group_seqs) = {len(seqs)} in len(prefix_len) + 1 "
                         f"steps, got {cu}")
    if any(not 0 <= b < nseq for b in seqs) or len(set(seqs)) != len(seqs):
        raise ValueError(f"shared_prefix: group_seqs must be distinct batch indices in [0, {nseq}), got {seqs}")
    if any(p <= 0 or p % int(block_size) for p in plen):
        raise ValueError(f"shared_prefix: every prefix_len must be a positive multiple of block_size {block_size}, got {plen}")
    return cu, seqs, plen


def _paged_kernels_ok(qkv, kc, d, block_size, quant=None, pro=None, shared_prefix=None):
    from ...framework.flags import flag

    dtype = qkv.dtype if pro is None else pro.dtype                      # the compute type: int32 qkv is dequantized to it
    cache_ok = kc.dtype == dtype or (quant is not None and kc.dtype in _KV8_DTYPES)
    # head_dim 64 has the decode, verify and prefill kernels over 16-bit caches only: no 8-bit caches, qkv prologue or shared prefix
    head_ok = d == 128 or (d == 64 and kc.dtype == dtype and pro is None and shared_prefix is None)
    return (qkv.is_cuda and kc.is_cuda and head_ok and dtype in (torch.float16, torch.bfloat16) and cache_ok
            and int(block_size) in _PREFILL_BLOCK_SIZES and flag("FLAGS_use_fused_kernels", True))


def _check_rope_positions(pro, max_pos):
    if pro is not None and pro.rope_cos is not None and max_pos >= pro.rope_cos.shape[0]:
        raise ValueError(f"block_multihead_attention: a new token sits at position {max_pos}, past the {pro.rope_cos.shape[0]} rows of rope_emb")


def block_attention(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size,
                    cache_k_quant_scales=None, cache_v_quant_scales=None, cache_k_dequant_scales=None, cache_v_dequant_scales=None,
                    use_dynamic_cachekv_quant=False, quant_round_type=1, quant_max_bound=127.0, quant_min_bound=-127.0, shared_prefix=None, *,
                    qkv_out_scale=None, qkv_bias=None, rope_emb=None, use_neox_style=False, out_shift=None, out_smooth=None, out_scale=-1,
                    compute_dtype="default", sliding_window=None):
    """qkv: [total_tokens, (H + 2*H_kv) * D] packed over the batch; caches [num_blocks, H_kv, block_size, D].

    A sequence prefills when seq_lens_encoder > 0 (a fresh prompt) or when it brings more than one token on top of seq_lens_decoder cached
    ones (a continuing chunk); it decodes when it brings exactly one token and seq_lens_encoder == 0.  A continuing chunk of 2 ..
    VERIFY_MAX tokens with now * (H / H_kv) <= 64 - the verify rows of speculative decoding - is a short chunk.

    CUDA path (head_dim 128 or 64, fp16 / bf16, block_size 16 / 32 / 64 / 128 / 256): the new K / V rows of EVERY sequence are scattered into the
    paged caches with one indexed write (block and row computed on the device from the block table - no per-token Python loop); decode
    sequences attend to their cache through `decode_attention_paged` (csrc/decode_attention.cu: one table lookup per cached row, split-K
    over the positions); all prefill sequences run in ONE launch of `attention_fwd_paged` (csrc/attention_sm100.cu): causal wgmma flash
    attention of each sequence's new tokens over its whole cached prefix, K / V read in place through the block table, q read and the
    output written in place at the tokens' rows; all short chunks run in ONE launch of `decode_attention_paged_multi`
    (csrc/decode_attention.cu: split-K over the cached positions, every query row of a KV head in one tensor-core tile, q and the output in
    place as for prefill).  The three row kinds are told apart with one host read.  Other block sizes and devices take
    `_block_attention_ref`; so does head_dim 64 with an 8-bit cache, the qkv prologue / out_scale or shared_prefix (those kernels are
    head_dim 128 only).

    int8 / float8_e4m3fn caches (static scales, see the module docstring): the new rows are quantized into the caches by one launch of
    `paged_kv_cache_write` (csrc/kv_cache_quant.cu), and the attention kernels read the 8-bit rows and dequantize them on the fly.

    shared_prefix = (cu_groups [G+1], group_seqs [n], prefix_len [G]), host lists or CPU int tensors: group g's members, the batch indices
    group_seqs[cu_groups[g]:cu_groups[g+1]], are decode rows whose first prefix_len[g] / block_size table entries are the same blocks
    (prefix_len a positive multiple of block_size, at most each member's cached length).  Their rows run in ONE launch pair of
    `decode_attention_paged_shared` (csrc/decode_attention.cu), which reads each group's prefix once per 64-row tile of members instead of
    once per member.  A grouped row that is not a decode row raises ValueError; a member whose table or length breaks the contract gets
    NaN rows (the device data is not read on the host).  Every other row takes its usual path.  None: no grouping.

    qkv prologue (each optional; T is the compute type: qkv's dtype, or compute_dtype 'bf16' / 'fp16' / 'fp32' for int32 qkv), applied to
    every new row in this order, each step rounded to T: int32 qkv is dequantized, float(qkv) * qkv_out_scale (fp32 [W]); qkv_bias (T [W])
    is added; rope_emb ([2, 1, S_rope, 1, R] cos, sin, read as fp32) rotates the Q and K heads at each token's position p: pairs (2i, 2i + 1)
    with R = D / 2, or with use_neox_style pairs (i, i + D / 2) with R = D (entries i >= D / 2 are not read), l' = l cos - r sin,
    r' = r cos + l sin, every product and sum rounded to fp32.  Decode rows read the table too (block_multihead_attention's rope_theta is
    not used).  The processed K / V rows are what the caches receive.  A float qkv gets its processed rows (q, k and v) written back in
    place; an int32 qkv is returned unchanged.  On the CUDA path the whole prologue and the cache write are ONE launch of
    `paged_kv_cache_write` (csrc/kv_cache_quant.cu), positions found on the device; a position >= S_rope raises ValueError before it,
    checked in the same host read that tells the row kinds apart.

    out_scale > 0: the output is quantized to int8 (quant_max_bound 127) or float8_e4m3fn (448) by one launch of `attention_out_quant`
    after the attention: y = max_bound * out_scale * o, rounded and clamped as the cache is (quant_round_type, bounds); out_shift /
    out_smooth (T [H * D], int8 output only) first replace o by ((o + shift) -> T) * smooth -> T.

    sliding_window = W (an int >= 1; None: off): local attention, the query at absolute position i sees key j iff i - W < j <= i.  Decode,
    verify and prefill rows go to the windowed instantiations of the paged kernels, which read only the window's cache rows and never read
    the table entries of blocks wholly below it (those blocks may have been released and reused).  Not combinable with shared_prefix."""
    sliding_window = _check_window(sliding_window, shared_prefix)
    qkv, kc, vc = _raw(qkv), _raw(key_cache), _raw(value_cache)
    nkv, d = kc.shape[1], kc.shape[3]
    quant = kv_quant_params(kc, vc, cache_k_quant_scales, cache_v_quant_scales, cache_k_dequant_scales, cache_v_dequant_scales,
                            use_dynamic_cachekv_quant, quant_round_type, quant_max_bound, quant_min_bound)
    nh = qkv.shape[1] // d - 2 * nkv
    pro = qkv_prologue_params(qkv, nh, nkv, d, qkv_out_scale, qkv_bias, rope_emb, use_neox_style, out_shift, out_smooth, out_scale, compute_dtype,
                              quant_round_type, quant_max_bound, quant_min_bound)
    if not _paged_kernels_ok(qkv, kc, d, block_size, quant, pro, shared_prefix):
        return _block_attention_ref(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables,
                                    block_size, quant=quant, shared_prefix=shared_prefix, prologue=pro, sliding_window=sliding_window)
    from ..._build import ext

    dev = qkv.device
    enc = _raw(seq_lens_encoder).reshape(-1).to(dev, torch.int64)
    dec = _raw(seq_lens_decoder).reshape(-1).to(dev, torch.int64)
    now = _raw(seq_lens_this_time).reshape(-1).to(dev, torch.int64)
    cu = _raw(cu_seqlens_q).reshape(-1).to(dev, torch.int64)
    bt = _raw(block_tables).to(dev, torch.int32).contiguous()
    nseq = now.numel()
    total_tokens = qkv.shape[0]
    past = torch.where(enc > 0, torch.zeros_like(dec), dec)                  # prefill starts at position 0, decode continues after the cache
    i32 = lambda t: t.to(torch.int32).contiguous()                          # noqa: E731
    dq = {} if quant is None else {"k_dequant_scales": quant.k_dequant, "v_dequant_scales": quant.v_dequant}
    if sliding_window is not None:
        dq["window"] = sliding_window
    if pro is not None:
        # ---- the row kinds and the last new position in one host read, then the prologue and the cache write in one launch
        kinds = _row_kinds(enc, now, nh, nkv, block_size, shared_prefix, torch.where(now > 0, past + now - 1, -1).max())
        _check_rope_positions(pro, kinds[-1])
        x = qkv if qkv.dtype != torch.int32 else torch.empty(qkv.shape, dtype=pro.dtype, device=dev)   # the processed rows
        ext().paged_kv_cache_write(qkv, kc, vc, i32(cu[:nseq + 1]), i32(enc), i32(dec), bt, *((quant.k_quant, quant.v_quant, quant.round_type,
                                   quant.max_bound, quant.min_bound) if quant is not None else (None, None, 1, 127.0, -127.0)),
                                   qkv_out=x if pro.has_prologue else None,
                                   qkv_out_scale=pro.qkv_out_scale, qkv_bias=pro.qkv_bias, rope_cos=pro.rope_cos, rope_sin=pro.rope_sin,
                                   neox=pro.neox)
    else:
        x = qkv
        if quant is None:
            # ---- scatter the new K / V rows into the paged caches (all sequences at once)
            rows = qkv.reshape(total_tokens, nh + 2 * nkv, d)
            k, v = rows[:, nh:nh + nkv], rows[:, nh + nkv:]
            tok = torch.arange(total_tokens, device=dev)
            seq_of = torch.bucketize(tok, cu[1:nseq + 1], right=True).clamp(max=nseq - 1)
            valid = tok < cu[nseq]
            pos = past[seq_of] + (tok - cu[seq_of])
            blk = bt.long()[seq_of, (pos // block_size).clamp(max=bt.shape[1] - 1)]
            off = pos % block_size
            sel = valid.nonzero().reshape(-1)
            kc[blk[sel], :, off[sel]] = k[sel]
            vc[blk[sel], :, off[sel]] = v[sel]
        else:
            # ---- quantize the new K / V rows into the 8-bit caches: one launch, rows read in place from qkv
            ext().paged_kv_cache_write(qkv.reshape(total_tokens, -1), kc, vc, i32(cu[:nseq + 1]), i32(enc), i32(dec), bt, quant.k_quant, quant.v_quant,
                                       quant.round_type, quant.max_bound, quant.min_bound)
        kinds = _row_kinds(enc, now, nh, nkv, block_size, shared_prefix)
    is_dec, is_ver, is_pre, groups, any_dec, any_ver, any_pre = kinds[:7]
    q = x.reshape(total_tokens, nh + 2 * nkv, d)[:, :nh]
    out = x.new_zeros((total_tokens, nh * d))
    scale = 1.0 / math.sqrt(d)
    if groups is not None:
        # ---- grouped decode rows: each group's prefix read once per tile of members, then every member's own keys
        ext().decode_attention_paged_shared(q, kc, vc, bt, i32(cu[:nseq]), i32(dec + 1), *(torch.tensor(v, dtype=torch.int32) for v in groups),
                                            scale, out, **dq)
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
    if pro is not None and pro.out_dtype is not None:
        # ---- output quantization: one launch over every row
        y = torch.empty(out.shape, dtype=pro.out_dtype, device=dev)
        ext().attention_out_quant(out, y, pro.out_scale, pro.out_shift, pro.out_smooth, pro.round_type, pro.max_bound, pro.min_bound)
        out = y
    return out.as_subclass(Tensor), qkv.as_subclass(Tensor), kc.as_subclass(Tensor), vc.as_subclass(Tensor)


def _check_window(sliding_window, shared_prefix):
    """sliding_window as an int >= 1, or None."""
    if sliding_window is None:
        return None
    if isinstance(sliding_window, bool) or not isinstance(sliding_window, int) or sliding_window < 1:
        raise ValueError(f"block_attention: sliding_window must be an int >= 1 or None, got {sliding_window!r}")
    if shared_prefix is not None:
        raise ValueError("block_attention: sliding_window cannot be combined with shared_prefix")
    return int(sliding_window)


def _row_kinds(enc, now, nh, nkv, block_size, shared_prefix, extra=None):
    """Splits block_attention's rows into decode / verify / prefill rows with ONE host read: (is_dec, is_ver, is_pre, shared-prefix groups or
    None, any_dec, any_ver, any_pre[, int(extra)]).  Grouped rows leave is_dec; a grouped row that is not a decode row raises ValueError."""
    nseq, dev = now.numel(), now.device
    is_dec = (now == 1) & (enc == 0)
    is_ver = (enc == 0) & (now >= 2) & (now <= min(VERIFY_MAX, 64 // (nh // nkv)))
    is_pre = (now > 0) & ~is_dec & ~is_ver
    groups = bad = None
    if shared_prefix is not None:
        groups = _shared_prefix_groups(shared_prefix, nseq, block_size)
        in_group = torch.zeros(nseq, dtype=torch.bool)
        in_group[groups[1]] = True
        in_group = in_group.pin_memory().to(dev, non_blocking=True)        # a pinned copy: the host does not wait for the stream
        bad = in_group & ~is_dec
        is_dec = is_dec & ~in_group
    flags = [is_dec.any(), is_ver.any(), is_pre.any()] + ([] if bad is None else [bad.any()])
    if extra is not None:
        flags = [f.long() for f in flags] + [extra]
    flags = torch.stack(flags).tolist()
    if shared_prefix is not None and flags.pop(3):
        raise ValueError("block_attention: shared_prefix groups may only hold decode rows (seq_lens_this_time 1, seq_lens_encoder 0)")
    return (is_dec, is_ver, is_pre, groups, *(bool(f) for f in flags[:3]), *(int(f) for f in flags[3:]))


def _block_attention_ref(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size,
                         cache_k_quant_scales=None, cache_v_quant_scales=None, cache_k_dequant_scales=None, cache_v_dequant_scales=None,
                         use_dynamic_cachekv_quant=False, quant_round_type=1, quant_max_bound=127.0, quant_min_bound=-127.0, quant=None,
                         shared_prefix=None, prologue=None, sliding_window=None, **prologue_args):
    """qkv: [total_tokens, (H + 2*H_kv) * D] packed over the batch; caches [num_blocks, H_kv, block_size, D].  `quant`: an already
    validated KVQuant (otherwise it is built from the scale / round / bound arguments).  `shared_prefix`: as in block_attention; its whole
    contract is checked here (ValueError on a violation), and it does not change the math.  `prologue`: an already validated QKVPrologue
    (otherwise it is built from block_attention's keyword arguments qkv_out_scale, qkv_bias, rope_emb, use_neox_style, out_shift,
    out_smooth, out_scale and compute_dtype in `prologue_args`), applied op by op in torch.  `sliding_window`: as in block_attention; only
    the cache rows of the window are read."""
    sliding_window = _check_window(sliding_window, shared_prefix)
    qkv, kc, vc = _raw(qkv), _raw(key_cache), _raw(value_cache)
    if quant is None:
        quant = kv_quant_params(kc, vc, cache_k_quant_scales, cache_v_quant_scales, cache_k_dequant_scales, cache_v_dequant_scales,
                                use_dynamic_cachekv_quant, quant_round_type, quant_max_bound, quant_min_bound)
    nkv, d = kc.shape[1], kc.shape[3]
    nh = qkv.shape[1] // d - 2 * nkv
    pro = prologue
    if pro is None:
        pro = qkv_prologue_params(qkv, nh, nkv, d, **prologue_args, quant_round_type=quant_round_type, quant_max_bound=quant_max_bound,
                                  quant_min_bound=quant_min_bound)
    enc, dec, now = _raw(seq_lens_encoder).reshape(-1).tolist(), _raw(seq_lens_decoder).reshape(-1).tolist(), _raw(seq_lens_this_time).reshape(-1).tolist()
    cu = _raw(cu_seqlens_q).reshape(-1).tolist()
    bt = _raw(block_tables)
    if shared_prefix is not None:
        _check_shared_prefix(shared_prefix, enc, dec, now, bt, block_size)
    x = qkv
    if pro is not None:
        starts = [0 if enc[b] > 0 else dec[b] for b in range(len(now))]
        _check_rope_positions(pro, max([starts[b] + now[b] - 1 for b in range(len(now)) if now[b] > 0], default=-1))
        if qkv.dtype == torch.int32:
            x = torch.zeros(qkv.shape, dtype=pro.dtype, device=qkv.device)
        if pro.has_prologue:
            for b in range(len(now)):
                if now[b] > 0:
                    pos = torch.arange(starts[b], starts[b] + now[b], device=qkv.device)
                    x[cu[b]:cu[b] + now[b]] = _prologue_ref(qkv[cu[b]:cu[b] + now[b]], pro, pos, nh, nkv, d)
    out = x.new_zeros((qkv.shape[0], nh * d))
    for b in range(len(now)):
        n = now[b]
        if n == 0:
            continue
        rows = x[cu[b]:cu[b] + n].reshape(n, nh + 2 * nkv, d)
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
        first = 0 if sliding_window is None else max(0, past - sliding_window + 1)   # the lowest key any new token sees
        b0 = first // block_size
        blks = bt[b, b0:nblk].long()
        K = kc[blks].permute(1, 0, 2, 3).reshape(nkv, (nblk - b0) * block_size, d)[:, first - b0 * block_size:total - b0 * block_size]
        V = vc[blks].permute(1, 0, 2, 3).reshape(nkv, (nblk - b0) * block_size, d)[:, first - b0 * block_size:total - b0 * block_size]
        if quant is not None:
            K, V = dequantize_kv(K, quant.k_dequant), dequantize_kv(V, quant.v_dequant)
        rep = nh // nkv
        K, V = K.repeat_interleave(rep, 0), V.repeat_interleave(rep, 0)
        s = torch.einsum("nhd,hsd->hns", q.float(), K.float()) / math.sqrt(d)
        qpos = torch.arange(past, total, device=qkv.device)[None, :, None]
        kpos = torch.arange(first, total, device=qkv.device)[None, None, :]
        hidden = kpos > qpos
        if sliding_window is not None:
            hidden = hidden | (kpos <= qpos - sliding_window)
        s = s.masked_fill(hidden, float("-inf"))
        o = torch.einsum("hns,hsd->nhd", torch.softmax(s, -1), V.float())
        out[cu[b]:cu[b] + n] = o.reshape(n, nh * d).to(out.dtype)
    if pro is not None and pro.out_dtype is not None:
        out = _out_quant_ref(out, pro)
    return out.as_subclass(Tensor), qkv.as_subclass(Tensor), kc.as_subclass(Tensor), vc.as_subclass(Tensor)


def _check_shared_prefix(shared_prefix, enc, dec, now, block_tables, block_size):
    """The full shared_prefix contract over host copies of the lengths and tables: ValueError on the first violation."""
    cu, seqs, plen = _shared_prefix_groups(shared_prefix, len(now), block_size)
    bt = block_tables.cpu()
    for g, p in enumerate(plen):
        idx = seqs[cu[g]:cu[g + 1]]
        nb = p // int(block_size)
        for b in idx:
            if now[b] != 1 or enc[b] != 0:
                raise ValueError(f"shared_prefix: sequence {b} is not a decode row (seq_lens_this_time {now[b]}, seq_lens_encoder {enc[b]})")
            if p > dec[b]:
                raise ValueError(f"shared_prefix: prefix_len {p} of group {g} exceeds the {dec[b]} cached tokens of sequence {b}")
            if nb > bt.shape[1] or not torch.equal(bt[b, :nb], bt[idx[0], :nb]):
                raise ValueError(f"shared_prefix: sequence {b} does not share the first {nb} blocks of group {g}")
