"""paddle.incubate.nn.functional (18 fused ops). Parity: python/paddle/incubate/nn/functional/*.py.
The hot ones (rms_norm, layer_norm, rope, swiglu, linear(+act), attention, softmax-CE) are the sm_100a kernels in
paddle_b200/csrc; the rest compose them."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as TF

from ....kernels import activation as KA
from ....kernels import attention as KAT
from ....kernels import gemm as KG
from ....kernels import norm as KN
from ....kernels import rope as KR
from ....tensor import Tensor


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


def _w(t):
    return t.as_subclass(Tensor) if isinstance(t, torch.Tensor) and not isinstance(t, Tensor) else t


def fused_rms_norm(x, norm_weight, norm_bias, epsilon, begin_norm_axis, bias=None, residual=None, quant_scale=-1, quant_round_type=0,
                   quant_max_bound=0, quant_min_bound=0):
    """Returns (out, residual_out) like the reference when residual is given, else out."""
    x = _raw(x)
    if bias is not None:
        x = x + _raw(bias)
    shape = x.shape
    x2 = x.reshape(-1, math.prod(shape[begin_norm_axis:]))
    if residual is not None:
        y, h = KN.rms_norm(x2, norm_weight, epsilon, norm_bias, residual=_raw(residual).reshape(x2.shape))
        out, res_out = _raw(y).reshape(shape), _raw(h).reshape(shape)
    else:
        out, res_out = _raw(KN.rms_norm(x2, norm_weight, epsilon, norm_bias)).reshape(shape), None
    if quant_scale > 0:
        out = torch.clamp(torch.round(out.float() * quant_max_bound * quant_scale), quant_min_bound, quant_max_bound).to(torch.int8)
    return (_w(out), _w(res_out)) if residual is not None else _w(out)


def fused_layer_norm(x, norm_weight, norm_bias, epsilon, residual_alpha=1.0, begin_norm_axis=1, bias=None, residual=None, quant_scale=-1,
                     quant_round_type=0, quant_max_bound=0, quant_min_bound=0):
    x = _raw(x)
    if bias is not None:
        x = x + _raw(bias)
    res_out = None
    if residual is not None:
        x = x + residual_alpha * _raw(residual)
        res_out = x
    shape = x.shape
    n = math.prod(shape[begin_norm_axis:])
    out = _raw(KN.layer_norm(x.reshape(-1, n), [n], None if norm_weight is None else _raw(norm_weight).reshape(-1),
                             None if norm_bias is None else _raw(norm_bias).reshape(-1), epsilon)).reshape(shape)
    return (_w(out), _w(res_out)) if residual is not None else _w(out)


def fused_rotary_position_embedding(q, k=None, v=None, sin=None, cos=None, position_ids=None, use_neox_rotary_style=True, time_major=False, rotary_emb_base=10000.0):
    """q/k/v: [B, S, H, D]. use_neox_rotary_style=True in the reference means *interleaved* pairs (GPT-NeoX "rotate every two")."""
    outs = []
    d = q.shape[-1]
    s = q.shape[0] if time_major else q.shape[1]
    if sin is None or cos is None:
        cos_t, sin_t = KR.rope_tables(s, d, rotary_emb_base, q.device)
    else:
        cos_t = _raw(cos).reshape(-1, d)[:, : d // 2].float() if not use_neox_rotary_style else _raw(cos).reshape(-1, d)[:, 0::2].float()
        sin_t = _raw(sin).reshape(-1, d)[:, : d // 2].float() if not use_neox_rotary_style else _raw(sin).reshape(-1, d)[:, 0::2].float()
    for t in (q, k, v):
        if t is None:
            outs.append(None)
            continue
        x = _raw(t).transpose(0, 1) if time_major else _raw(t)
        y = _raw(KR.apply_rope(x.contiguous(), cos_t, sin_t, position_ids, neox=not use_neox_rotary_style))
        outs.append(_w(y.transpose(0, 1) if time_major else y))
    return tuple(outs)


def swiglu(x, y=None, name=None):
    return KA.swiglu(x, y)


def fused_matmul_bias(x, y, bias=None, transpose_x=False, transpose_y=False, name=None):
    x2 = _raw(x)
    if not transpose_x and not transpose_y and x2.dim() >= 2 and _raw(y).dim() == 2:
        return KG.linear(x2, y, bias)
    out = KG.matmul(x2, y, transpose_x, transpose_y)
    return out + bias if bias is not None else out


def fused_linear(x, weight, bias=None, transpose_weight=False, name=None):
    return fused_matmul_bias(x, weight, bias, False, transpose_weight)


def fused_linear_activation(x, y, bias, trans_x=False, trans_y=False, activation=None):
    out = fused_matmul_bias(x, y, bias, trans_x, trans_y)
    if activation in (None, "none"):
        return out
    return {"gelu": TF.gelu, "relu": torch.relu}[activation](out)


def _fused_ew_ok(x, *others):
    """CUDA tensors of one 16-bit / fp32 dtype whose last dimension fills whole 16-byte vectors: csrc/fused_dropout.cu applies."""
    from ....framework.flags import flag

    if not (isinstance(x, torch.Tensor) and x.is_cuda and flag("FLAGS_use_fused_kernels", True)) or x.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        return False
    vec = 16 // x.element_size()
    if x.dim() < 1 or x.shape[-1] % vec or x.numel() == 0:
        return False
    return all(o is None or (o.is_cuda and o.dtype == x.dtype) for o in others)


def fused_bias_act(x, bias=None, dequant_scales=None, shift=None, smooth=None, act_method="gelu", compute_dtype="default", quant_scale=-1,
                   quant_round_type=0, quant_max_bound=0, quant_min_bound=0):
    x = _raw(x)
    b = None if bias is None else _raw(bias)
    act_id = {"gelu": 0, "relu": 1, "silu": 2, "swish": 2, "geglu": 0, "swiglu": 2}.get(act_method)
    gated = act_method in ("swiglu", "geglu")
    if dequant_scales is None and shift is None and smooth is None and quant_scale <= 0 and act_id is not None and _fused_ew_ok(x, b) and not (x.requires_grad and torch.is_grad_enabled()) \
            and (not gated or (x.shape[-1] // 2) % (16 // x.element_size()) == 0) and (b is None or b.numel() == x.shape[-1]):
        from ...._build import ext

        return _w(ext().bias_act(x.contiguous(), None if b is None else b.contiguous(), act_id, gated))     # one pass: csrc/fused_dropout.cu
    if dequant_scales is not None:
        x = x.float() * _raw(dequant_scales)
    if bias is not None:
        x = x + _raw(bias)
    if act_method in ("swiglu",):
        out = _raw(KA.swiglu(x))
    elif act_method == "geglu":
        a, b = x.chunk(2, -1)
        out = TF.gelu(a) * b
    else:
        out = {"gelu": TF.gelu, "relu": torch.relu, "silu": TF.silu, "swish": TF.silu}[act_method](x)
    if shift is not None:
        out = out + _raw(shift)
    if smooth is not None:
        out = out * _raw(smooth)
    if quant_scale > 0:
        out = torch.clamp(torch.round(out.float() * quant_max_bound * quant_scale), quant_min_bound, quant_max_bound).to(torch.int8)
    return _w(out)


class _BiasDropoutAdd(torch.autograd.Function):
    """out = dropout(x + bias) + y in one kernel; the byte mask is the only thing saved.  Philox counter: (seed, offset) from the framework
    generator, advanced per call so that successive calls never reuse a stream position."""

    @staticmethod
    def forward(ctx, x, bias, y, p, upscale):
        from ...._build import ext

        # the device generator owns the Philox position: take (seed, offset) from it and advance it by what one vector stream may draw
        # (two uniform4 = 8 values), exactly like a native dropout would - re-seeding replays the same masks
        gen = torch.cuda.default_generators[x.device.index if x.device.index is not None else torch.cuda.current_device()]
        seed = int(gen.initial_seed()) & 0x7FFFFFFFFFFFFFFF
        offset = int(gen.get_offset())
        gen.set_offset(offset + 8)
        out, mask = ext().bias_dropout_add(x.contiguous(), None if bias is None else bias.contiguous(), None if y is None else y.contiguous(), float(p), bool(upscale), seed, offset)
        ctx.save_for_backward(mask)
        ctx.p, ctx.upscale, ctx.has_bias, ctx.has_y = float(p), bool(upscale), bias is not None, y is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        from ...._build import ext

        (mask,) = ctx.saved_tensors
        dx = ext().dropout_bwd(dout.contiguous(), mask, ctx.p, ctx.upscale)
        dbias = dx.reshape(-1, dx.shape[-1]).sum(0) if ctx.has_bias else None
        return dx, dbias, (dout if ctx.has_y else None), None, None


def fused_dropout_add(x, y, p=0.5, training=True, mode="upscale_in_train", name=None):
    from ....nn import functional as F

    xr, yr = _raw(x), _raw(y)
    if training and 0.0 < p < 1.0 and _fused_ew_ok(xr, yr) and xr.shape == yr.shape:
        return _w(_BiasDropoutAdd.apply(xr, None, yr, p, mode == "upscale_in_train"))
    return F.dropout(x, p, training=training, mode=mode) + y


def fused_bias_dropout_residual_layer_norm(x, residual, bias=None, ln_scale=None, ln_bias=None, dropout_rate=0.5, ln_epsilon=1e-5, training=True,
                                           mode="upscale_in_train", name=None):
    from ....nn import functional as F

    xr, rr, br = _raw(x), _raw(residual), (None if bias is None else _raw(bias))
    if training and 0.0 < dropout_rate < 1.0 and _fused_ew_ok(xr, rr, br) and xr.shape == rr.shape and (br is None or br.numel() == xr.shape[-1]):
        h = _w(_BiasDropoutAdd.apply(xr, br, rr, dropout_rate, mode == "upscale_in_train"))      # bias + dropout + residual: one pass
        return F.layer_norm(h, [h.shape[-1]], ln_scale, ln_bias, ln_epsilon)                      # fused LayerNorm kernel (csrc/norm.cu)
    h = x if bias is None else x + bias
    h = F.dropout(h, dropout_rate, training=training, mode=mode) + residual
    return F.layer_norm(h, [h.shape[-1]], ln_scale, ln_bias, ln_epsilon)


def fused_dot_product_attention(query, key, value, attn_mask=None, dropout_p=0.0, is_causal=False, scaling_factor=None, training=True, name=None, dropout_prob=None):
    q, k, v = query, key, value
    dropout_prob = dropout_p if dropout_prob is None else dropout_prob
    return KAT.attention(q, k, v, attn_mask, dropout_prob if training else 0.0, is_causal, scaling_factor)


def fused_multi_head_attention(x, qkv_weight, linear_weight, pre_layer_norm=False, pre_ln_scale=None, pre_ln_bias=None, ln_scale=None, ln_bias=None,
                               pre_ln_epsilon=1e-05, qkv_bias=None, linear_bias=None, cache_kv=None, attn_mask=None, dropout_rate=0.5,
                               attn_dropout_rate=0.5, ln_epsilon=1e-05, training=True, mode="upscale_in_train", ring_id=-1, add_residual=True,
                               num_heads=-1, transpose_qkv_wb=False, name=None):
    """Parity: incubate/nn/functional/fused_transformer.py:fused_multi_head_attention. qkv_weight: [3, H, D, E] (or [E, 3E] if transpose_qkv_wb)."""
    from ....nn import functional as F

    xr = _raw(x)
    residual = xr
    h = _raw(F.layer_norm(x, [xr.shape[-1]], pre_ln_scale, pre_ln_bias, pre_ln_epsilon)) if pre_layer_norm else xr
    qw = _raw(qkv_weight)
    if transpose_qkv_wb:
        nh = num_heads
        qkv = h @ qw
        if qkv_bias is not None:
            qkv = qkv + _raw(qkv_bias)
        b, s, _ = qkv.shape
        q, k, v = qkv.reshape(b, s, 3, nh, -1).unbind(2)
    else:
        _, nh, hd, e = qw.shape
        qkv = torch.einsum("bse,thde->bsthd", h, qw)
        if qkv_bias is not None:
            qkv = qkv + _raw(qkv_bias).reshape(1, 1, 3, nh, hd)
        q, k, v = qkv.unbind(2)
    cache_out = None
    if cache_kv is not None:
        ck = _raw(cache_kv)  # [2, B, H, S_cache, D]
        k = torch.cat([ck[0].transpose(1, 2), k], 1)
        v = torch.cat([ck[1].transpose(1, 2), v], 1)
        cache_out = torch.stack([k.transpose(1, 2), v.transpose(1, 2)])
    mask = None if attn_mask is None else _raw(attn_mask)
    o = _raw(KAT.attention(q, k, v, mask, attn_dropout_rate if training else 0.0, False, None))
    o = o.reshape(o.shape[0], o.shape[1], -1) @ _raw(linear_weight)
    if linear_bias is not None:
        o = o + _raw(linear_bias)
    o = _raw(F.dropout(_w(o), dropout_rate, training=training, mode=mode))
    if add_residual:
        o = o + residual
    if not pre_layer_norm:
        o = _raw(F.layer_norm(_w(o), [o.shape[-1]], ln_scale, ln_bias, ln_epsilon))
    return (_w(o), _w(cache_out)) if cache_kv is not None else _w(o)


def fused_feedforward(x, linear1_weight, linear2_weight, linear1_bias=None, linear2_bias=None, ln1_scale=None, ln1_bias=None, ln2_scale=None,
                      ln2_bias=None, dropout1_rate=0.5, dropout2_rate=0.5, activation="relu", ln1_epsilon=1e-5, ln2_epsilon=1e-5,
                      pre_layer_norm=False, training=True, mode="upscale_in_train", ring_id=-1, add_residual=True, name=None):
    from ....nn import functional as F

    residual = x
    h = F.layer_norm(x, [x.shape[-1]], ln1_scale, ln1_bias, ln1_epsilon) if pre_layer_norm else x
    h = F.linear(h, linear1_weight, linear1_bias)
    h = getattr(F, activation)(h)
    h = F.dropout(h, dropout1_rate, training=training, mode=mode)
    h = F.linear(h, linear2_weight, linear2_bias)
    h = F.dropout(h, dropout2_rate, training=training, mode=mode)
    if add_residual:
        h = h + residual
    if not pre_layer_norm:
        h = F.layer_norm(h, [h.shape[-1]], ln2_scale, ln2_bias, ln2_epsilon)
    return h


def masked_multihead_attention(x, cache_kv=None, bias=None, src_mask=None, cum_offsets=None, sequence_lengths=None, rotary_tensor=None,
                               beam_cache_offset=None, qkv_out_scale=None, out_shift=None, out_smooth=None, seq_len=1, rotary_emb_dims=0,
                               use_neox_rotary_style=False, compute_dtype="default", out_scale=-1, quant_round_type=1, quant_max_bound=127.0,
                               quant_min_bound=-127.0):
    """Single-token decode attention against a KV cache [2, B, H, S_max, D]. Parity: masked_multihead_attention.py."""
    xr, ck = _raw(x), _raw(cache_kv)
    _, b, nh, smax, hd = ck.shape
    qkv = xr.reshape(b, 3, nh, hd)
    if bias is not None:
        qkv = qkv + _raw(bias).reshape(1, 3, nh, hd)
    q, k, v = qkv.unbind(1)
    lens = _raw(sequence_lengths).reshape(-1).long() if sequence_lengths is not None else torch.full((b,), seq_len - 1 if seq_len > 0 else 0, device=xr.device, dtype=torch.long)
    bi = torch.arange(b, device=xr.device)
    ck[0, bi, :, lens] = k.to(ck.dtype)
    ck[1, bi, :, lens] = v.to(ck.dtype)
    if src_mask is None and xr.is_cuda and hd == 128 and ck.dtype in (torch.bfloat16, torch.float16) and ck.is_contiguous():
        # HBM-bound split-KV decode kernel (csrc/decode_attention.cu): each cached row is read once with 16-byte loads
        from ...._build import ext

        out = ext().decode_attention(q.to(ck.dtype).contiguous(), ck[0], ck[1], (lens + 1).to(torch.int32).contiguous(), 1.0 / math.sqrt(hd))
        return _w(out.reshape(b, nh * hd).to(xr.dtype)), _w(ck)
    scores = torch.einsum("bhd,bhsd->bhs", q.float(), ck[0].float()) / math.sqrt(hd)
    pos = torch.arange(smax, device=xr.device)[None, None]
    scores = scores.masked_fill(pos > lens[:, None, None], float("-inf"))
    if src_mask is not None:
        scores = scores + _raw(src_mask).reshape(b, 1, -1)[..., :smax].float()
    p = torch.softmax(scores, -1)
    out = torch.einsum("bhs,bhsd->bhd", p, ck[1].float()).reshape(b, nh * hd).to(xr.dtype)
    return _w(out), _w(ck)


def variable_length_memory_efficient_attention(query, key, value, seq_lens, kv_seq_lens, mask=None, scale=None, causal=False, pre_cache_length=0):
    """q/k/v [B, H, S, D] with per-batch valid lengths."""
    q, k, v = _raw(query), _raw(key), _raw(value)
    b, h, sq, d = q.shape
    sk = k.shape[2]
    ql, kl = _raw(seq_lens).reshape(-1), _raw(kv_seq_lens).reshape(-1)
    scale = scale or 1.0 / math.sqrt(d)
    s = (q.float() @ k.float().transpose(-1, -2)) * scale
    valid = (torch.arange(sk, device=q.device)[None, None, None] < kl.reshape(b, 1, 1, 1))
    if causal:
        valid = valid & (torch.arange(sk, device=q.device)[None, None, None] <= torch.arange(sq, device=q.device)[None, None, :, None] + pre_cache_length)
    if mask is not None:
        s = s + _raw(mask).float()
    s = s.masked_fill(~valid, float("-inf"))
    o = torch.softmax(s, -1).nan_to_num(0.0) @ v.float()
    o = o * (torch.arange(sq, device=q.device)[None, None, :, None] < ql.reshape(b, 1, 1, 1))
    return _w(o.to(q.dtype))


def block_multihead_attention(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, padding_offsets, cum_offsets,
                              cu_seqlens_q, cu_seqlens_k, block_tables, pre_key_cache=None, pre_value_cache=None, cache_k_quant_scales=None,
                              cache_v_quant_scales=None, cache_k_dequant_scales=None, cache_v_dequant_scales=None, qkv_out_scale=None, qkv_bias=None,
                              out_shift=None, out_smooth=None, max_enc_len_this_time=None, max_dec_len_this_time=None, rope_emb=None, mask=None,
                              tgt_mask=None, max_seq_len=-1, block_size=64, use_neox_style=False, use_dynamic_cachekv_quant=False, quant_round_type=1,
                              quant_max_bound=127.0, quant_min_bound=-127.0, out_scale=-1, compute_dtype="default", rope_theta=10000.0):
    """Paged-KV attention (prefill + decode). Parity: block_multihead_attention.py. key/value_cache: [num_blocks, H_kv, block_size, D].

    int8 / float8_e4m3fn caches take static per-KV-head cache_{k,v}_{quant,dequant}_scales (fp32 [H_kv]) with quant_round_type and the
    quant bounds (see incubate.nn.paged_attention).  Dynamic cache quantization raises NotImplementedError; scales with a 16-bit cache, or an
    8-bit cache without them, raise ValueError.  The pre-caches, rope_emb, masks, qkv_out_scale / bias, out_shift / smooth and out_scale
    are not applied."""
    from ....incubate.nn.paged_attention import block_attention

    return block_attention(qkv, key_cache, value_cache, seq_lens_encoder, seq_lens_decoder, seq_lens_this_time, cu_seqlens_q, block_tables, block_size,
                           cache_k_quant_scales, cache_v_quant_scales, cache_k_dequant_scales, cache_v_dequant_scales, use_dynamic_cachekv_quant,
                           quant_round_type, quant_max_bound, quant_min_bound)


def blha_get_max_len(seq_lens_encoder, seq_lens_decoder, batch_size):
    return _w(_raw(seq_lens_encoder).max().reshape(1)), _w(_raw(seq_lens_decoder).max().reshape(1))


def fused_gate_attention(query, key=None, query_weight=None, key_weight=None, value_weight=None, qkv_weight=None, gate_linear_weight=None,
                         gate_linear_bias=None, out_linear_weight=None, out_linear_bias=None, nonbatched_bias=None, attn_mask=None,
                         has_gating=True, merge_qkv=True, use_flash_attn=False):
    """AlphaFold-style gated attention. query [B, M, R, E]."""
    q_in = _raw(query)
    if merge_qkv:
        qw = _raw(qkv_weight)  # [3, H, D, E]
        qkv = torch.einsum("bmre,thde->tbmrhd", q_in, qw)
        q, k, v = qkv[0], qkv[1], qkv[2]
    else:
        k_in = _raw(key) if key is not None else q_in
        q = torch.einsum("bmre,ehd->bmrhd", q_in, _raw(query_weight))
        k = torch.einsum("bmre,ehd->bmrhd", k_in, _raw(key_weight))
        v = torch.einsum("bmre,ehd->bmrhd", k_in, _raw(value_weight))
    d = q.shape[-1]
    s = torch.einsum("bmqhd,bmkhd->bmhqk", q, k) / math.sqrt(d)
    if nonbatched_bias is not None:
        s = s + _raw(nonbatched_bias).unsqueeze(1)
    if attn_mask is not None:
        s = s + _raw(attn_mask)
    o = torch.einsum("bmhqk,bmkhd->bmqhd", torch.softmax(s, -1), v)
    if has_gating:
        g = torch.sigmoid(torch.einsum("bmre,ehd->bmrhd", q_in, _raw(gate_linear_weight)) + _raw(gate_linear_bias))
        o = o * g
    out = torch.einsum("bmrhd,hde->bmre", o, _raw(out_linear_weight)) + _raw(out_linear_bias)
    return _w(out)


def fused_moe(x, gate_weight, ffn1_weight, ffn2_weight, ffn1_bias=None, ffn1_scale=None, ffn2_bias=None, ffn2_scale=None, quant_method="None",
              moe_topk=2, norm_topk_prob=True, group_moe=False):
    """Token-choice top-k MoE FFN (SwiGLU experts). Parity: incubate/nn/functional/fused_moe.py."""
    from ....incubate.moe import moe_ffn

    return moe_ffn(x, gate_weight, ffn1_weight, ffn1_bias, ffn2_weight, ffn2_bias, moe_topk, norm_topk_prob)


__all__ = ["fused_multi_head_attention", "fused_feedforward", "fused_multi_transformer", "fused_matmul_bias", "fused_linear", "fused_linear_activation",
           "fused_bias_dropout_residual_layer_norm", "fused_dropout_add", "fused_rotary_position_embedding", "variable_length_memory_efficient_attention",
           "fused_rms_norm", "fused_layer_norm", "fused_bias_act", "masked_multihead_attention", "blha_get_max_len", "block_multihead_attention",
           "swiglu", "fused_dot_product_attention", "fused_gate_attention", "fused_moe"]


def fused_multi_transformer(x, ln_scales, ln_biases, qkv_weights, qkv_biases, linear_weights, linear_biases, ffn_ln_scales, ffn_ln_biases,
                            ffn1_weights, ffn1_biases, ffn2_weights, ffn2_biases, pre_layer_norm=True, epsilon=1e-05, residual_alpha=1.0, cache_kvs=None,
                            beam_offset=None, pre_caches=None, seq_lens=None, rotary_embs=None, time_step=None, attn_mask=None, dropout_rate=0.0,
                            rotary_emb_dims=0, activation="gelu", training=False, mode="upscale_in_train", trans_qkvw=True, ring_id=-1,
                            norm_type="layernorm", use_neox_rotary_style=False, gqa_group_size=-1, name=None):
    """Stack of fused decoder layers with optional KV caches. Parity: fused_transformer.py:fused_multi_transformer."""
    from ....nn import functional as F

    h = x
    new_caches = []
    for i in range(len(qkv_weights)):
        residual = h
        y = F.layer_norm(h, [h.shape[-1]], ln_scales[i], ln_biases[i], epsilon) if pre_layer_norm else h
        qw = _raw(qkv_weights[i])
        if trans_qkvw:       # [3, H, D, E]
            _, nh, hd, e = qw.shape
            qkv = torch.einsum("bse,thde->bsthd", _raw(y), qw)
        else:                # [E, 3, H, D]
            e, _, nh, hd = qw.shape
            qkv = torch.einsum("bse,ethd->bsthd", _raw(y), qw)
        if qkv_biases is not None and qkv_biases[i] is not None:
            qkv = qkv + _raw(qkv_biases[i]).reshape(1, 1, 3, nh, hd)
        q, k, v = qkv.unbind(2)
        if rotary_embs is not None and rotary_emb_dims > 0:
            re = _raw(rotary_embs)  # [2, B, 1, S, D]
            cos_t, sin_t = re[0, 0, 0, :, : hd // 2].float(), re[1, 0, 0, :, : hd // 2].float()
            pos = None if time_step is None else (torch.zeros(q.shape[0], q.shape[1], dtype=torch.long, device=q.device) + int(_raw(time_step).item()))
            q = _raw(KR.apply_rope(q.contiguous(), cos_t, sin_t, pos, neox=True))
            k = _raw(KR.apply_rope(k.contiguous(), cos_t, sin_t, pos, neox=True))
        causal = False
        if cache_kvs is not None:
            ck = _raw(cache_kvs[i])  # [2, B, H, S_max, D]
            if time_step is None:    # prefill: write the prompt
                s = k.shape[1]
                ck[0, :, :, :s] = k.transpose(1, 2)
                ck[1, :, :, :s] = v.transpose(1, 2)
                causal = attn_mask is None
            else:
                t = int(_raw(time_step).item())
                ck[0, :, :, t] = k[:, 0]
                ck[1, :, :, t] = v[:, 0]
                k, v = ck[0, :, :, : t + 1].transpose(1, 2), ck[1, :, :, : t + 1].transpose(1, 2)
            new_caches.append(_w(ck))
        o = _raw(KAT.attention(q, k, v, None if attn_mask is None else _raw(attn_mask), 0.0, causal, None))
        o = o.reshape(o.shape[0], o.shape[1], -1) @ _raw(linear_weights[i])
        if linear_biases is not None and linear_biases[i] is not None:
            o = o + _raw(linear_biases[i])
        h = _w(o) + residual
        if not pre_layer_norm:
            h = F.layer_norm(h, [h.shape[-1]], ln_scales[i], ln_biases[i], epsilon)
        residual = h
        y = F.layer_norm(h, [h.shape[-1]], ffn_ln_scales[i], ffn_ln_biases[i], epsilon) if pre_layer_norm else h
        y = F.linear(y, ffn1_weights[i], None if ffn1_biases is None else ffn1_biases[i])
        y = getattr(F, activation)(y)
        y = F.linear(y, ffn2_weights[i], None if ffn2_biases is None else ffn2_biases[i])
        h = y + residual
        if not pre_layer_norm:
            h = F.layer_norm(h, [h.shape[-1]], ffn_ln_scales[i], ffn_ln_biases[i], epsilon)
    return (h, new_caches) if cache_kvs is not None else h


from ....framework.recording import make_recordable as _make_recordable  # noqa: E402

# Static-graph recording: these functions work on raw tensors (fast paths straight into the kernels), which the op tape cannot see; each public entry
# point is therefore recorded as ONE node.  Outside a program_guard the wrapper is a single `is None` test.
_make_recordable(globals(), __all__)
