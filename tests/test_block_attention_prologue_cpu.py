"""block_multihead_attention's qkv prologue (int32 dequantization, qkv_bias, rope_emb) and out_scale output quantization on the CPU path:
against an independent per-token loop, against the models' own rotary (kernels.rope), int32 against the float path, the output rounding
rules, and the argument errors."""
import pytest
import torch

from paddle_b200.incubate.nn import functional as IF
from paddle_b200.incubate.nn import paged_attention as PA
from paddle_b200.kernels import rope as R

D = 128
THETA = 10000.0
# (enc, dec, now): a fresh prompt, a continuing chunk longer than VERIFY_MAX, verify rows, and two decode rows
SPECS = [(21, 0, 21), (0, 30, 19), (0, 50, 4), (0, 40, 1), (0, 70, 1)]
BOUND = {torch.int8: 127.0, torch.float8_e4m3fn: 448.0}


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) else t


def mixed_batch(specs, nh, nkv, bs, dtype, kv=None, seed=0, device="cpu"):
    """Packed qkv [T, (H + 2 Hkv) * D] of `dtype`, random caches of `dtype` (or 8-bit `kv` with static scales), shuffled block tables.
    Returns qkv, kc, vc, args (enc, dec, now, cu, bt, bs) and the cache quantization keyword arguments."""
    g = torch.Generator().manual_seed(seed)
    enc = torch.tensor([s[0] for s in specs], dtype=torch.int32)
    dec = torch.tensor([s[1] for s in specs], dtype=torch.int32)
    now = torch.tensor([s[2] for s in specs], dtype=torch.int32)
    cu = torch.zeros(len(specs) + 1, dtype=torch.int32)
    cu[1:] = torch.cumsum(now, 0)
    need = [((0 if e > 0 else d) + n + bs - 1) // bs for e, d, n in specs]
    max_blocks = max(need) + 1
    nblocks = sum(need) + 3
    perm = torch.randperm(nblocks, generator=g)
    bt = torch.full((len(specs), max_blocks), int(perm[-1]), dtype=torch.int32)
    nxt = 0
    for i, k in enumerate(need):
        bt[i, :k] = perm[nxt:nxt + k]
        nxt += k
    qkv = (torch.randn(int(cu[-1]), (nh + 2 * nkv) * D, generator=g) * 0.7).to(dtype)
    quant = {}
    if kv is None:
        kc = (torch.randn(nblocks, nkv, bs, D, generator=g) * 0.7).to(dtype)
        vc = (torch.randn(nblocks, nkv, bs, D, generator=g) * 0.7).to(dtype)
    else:
        bound = BOUND[kv]
        kc = (torch.randn(nblocks, nkv, bs, D, generator=g) * bound / 4).clamp(-bound, bound).to(kv)
        vc = (torch.randn(nblocks, nkv, bs, D, generator=g) * bound / 4).clamp(-bound, bound).to(kv)
        qs = torch.full((nkv,), 0.25)
        quant = dict(cache_k_quant_scales=qs, cache_v_quant_scales=qs * 0.5, cache_k_dequant_scales=1.0 / (bound * qs),
                     cache_v_dequant_scales=2.0 / (bound * qs), quant_max_bound=bound, quant_min_bound=-bound)
    args = tuple(t.to(device) for t in (enc, dec, now, cu, bt)) + (bs,)
    quant = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in quant.items()}
    return qkv.to(device), kc.to(device), vc.to(device), args, quant


def rope_emb_from_tables(npos, neox, device="cpu"):
    """rope_emb [2, 1, npos, 1, R] from the models' tables: R = D / 2, or the table twice along the last axis (R = D) for neox."""
    cos, sin = R.rope_tables(npos, D, THETA, device=device)
    if neox:
        cos, sin = torch.cat([cos, cos], -1), torch.cat([sin, sin], -1)
    return torch.stack([cos, sin])[:, None, :, None, :].contiguous()


def call(qkv, kc, vc, args, **kw):
    """block_multihead_attention on the (enc, dec, now, cu, bt, bs) batch layout of mixed_batch."""
    enc, dec, now, cu, bt, bs = args
    out = IF.block_multihead_attention(qkv, kc, vc, enc, dec, now, None, None, cu, None, bt, block_size=bs, **kw)
    return tuple(_raw(t) for t in out)


def _process_per_token(qkv, args, nh, nkv, neox, bias=None, col_scale=None, dtype=None):
    """The prologue written out token by token: dequantize, add the bias, rotate the Q and K heads at the token's position with angles
    p * THETA^(-2i / D) computed here."""
    enc, dec, now, cu, _, _ = args
    dtype = dtype or qkv.dtype
    out = torch.zeros(qkv.shape, dtype=dtype)
    inv = 1.0 / (THETA ** (torch.arange(0, D, 2, dtype=torch.float32) / D))
    for b in range(len(now)):
        start = 0 if int(enc[b]) > 0 else int(dec[b])
        for t in range(int(now[b])):
            row = qkv[int(cu[b]) + t]
            x = (row.float() * col_scale).to(dtype) if col_scale is not None else row
            if bias is not None:
                x = x + bias
            heads = x.reshape(nh + 2 * nkv, D).clone()
            ang = torch.tensor(float(start + t), dtype=torch.float32) * inv
            c, s = ang.cos(), ang.sin()
            qk = heads[:nh + nkv].float()
            if neox:
                lo, hi = qk[:, :D // 2], qk[:, D // 2:]
                heads[:nh + nkv] = torch.cat([lo * c - hi * s, hi * c + lo * s], 1).to(dtype)
            else:
                ev, od = qk[:, 0::2], qk[:, 1::2]
                heads[:nh + nkv] = torch.stack([ev * c - od * s, od * c + ev * s], -1).reshape(nh + nkv, D).to(dtype)
            out[int(cu[b]) + t] = heads.reshape(-1)
    return out


def _bits(t):
    return t.view(torch.uint8) if t.dtype == torch.float8_e4m3fn else t


@pytest.mark.parametrize("neox", [False, True])
@pytest.mark.parametrize("heads", [(32, 8), (32, 32)])
@pytest.mark.parametrize("kv", [None, torch.int8, torch.float8_e4m3fn])
def test_rope_and_bias_equal_a_prologue_free_call_on_processed_rows(kv, heads, neox):
    nh, nkv = heads
    qkv, kc, vc, args, quant = mixed_batch(SPECS, nh, nkv, 16, torch.bfloat16, kv, seed=nh + nkv)
    bias = (torch.randn(qkv.shape[1], generator=torch.Generator().manual_seed(7)) * 0.3).to(torch.bfloat16)
    rope_emb = rope_emb_from_tables(128, neox)
    got = call(qkv.clone(), kc.clone(), vc.clone(), args, qkv_bias=bias, rope_emb=rope_emb, use_neox_style=neox, rope_theta=THETA, **quant)
    rows = _process_per_token(qkv, args, nh, nkv, neox, bias=bias)
    want = call(rows.clone(), kc.clone(), vc.clone(), args, **quant)
    assert torch.equal(got[1], rows)                                       # float qkv: the processed rows, written back in place
    for a, b in zip(got[:1] + got[2:], want[:1] + want[2:]):
        assert torch.equal(_bits(a), _bits(b))
    assert not torch.equal(rows, qkv)


@pytest.mark.parametrize("heads", [(32, 8), (32, 32)])
def test_neox_rope_matches_the_models_rotary(heads):
    nh, nkv = heads
    qkv, kc, vc, args, _ = mixed_batch(SPECS, nh, nkv, 16, torch.bfloat16, seed=1)
    got = call(qkv.clone(), kc.clone(), vc.clone(), args, rope_emb=rope_emb_from_tables(100, True), use_neox_style=True)
    enc, dec, now, cu, _, _ = args
    cos, sin = R.rope_tables(100, D, THETA)
    rows = qkv.clone()
    for b in range(len(now)):
        start = 0 if int(enc[b]) > 0 else int(dec[b])
        seg = rows[int(cu[b]):int(cu[b + 1])][None]                         # [1, n, W]
        pos = torch.arange(start, start + int(now[b]))[None]
        rows[int(cu[b]):int(cu[b + 1])] = _raw(R.apply_rope_packed(seg, cos, sin, nh + nkv, nh + 2 * nkv, D, position_ids=pos, neox=True))[0]
    want = call(rows.clone(), kc.clone(), vc.clone(), args)
    err = ((got[0].float() - want[0].float()).norm() / want[0].float().norm()).item()
    assert err < 2e-2, err
    assert ((got[1].float() - rows.float()).abs().max() <= 2 ** -7 * rows.float().abs().max())


@pytest.mark.parametrize("kv", [None, torch.int8])
@pytest.mark.parametrize("compute_dtype,dtype", [("bf16", torch.bfloat16), ("fp16", torch.float16), ("fp32", torch.float32)])
def test_int32_qkv_equals_the_float_path_on_dequantized_rows(compute_dtype, dtype, kv):
    nh, nkv = 8, 2
    _, kc, vc, args, quant = mixed_batch(SPECS, nh, nkv, 16, dtype, kv, seed=2)
    g = torch.Generator().manual_seed(3)
    w = (nh + 2 * nkv) * D
    qkv = torch.randint(-3000, 3000, (int(args[3][-1]), w), generator=g, dtype=torch.int32)
    col_scale = torch.rand(w, generator=g) * 4e-4
    bias = (torch.randn(w, generator=g) * 0.2).to(dtype)
    pro = dict(qkv_bias=bias, rope_emb=rope_emb_from_tables(128, False), **quant)
    got = call(qkv.clone(), kc.clone(), vc.clone(), args, qkv_out_scale=col_scale, compute_dtype=compute_dtype, **pro)
    rows = (qkv.float() * col_scale).to(dtype)
    want = call(rows, kc.clone(), vc.clone(), args, **pro)
    assert torch.equal(got[1], qkv)                                        # int32 qkv comes back unchanged
    for a, b in zip(got[:1] + got[2:], want[:1] + want[2:]):
        assert a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))
    proc = _process_per_token(qkv, args, nh, nkv, False, bias=bias, col_scale=col_scale, dtype=dtype)
    assert torch.equal(want[1], proc)


def _out_quant(o, out_scale, **kw):
    """block_attention's epilogue on fixed attention output o [T, H * D]: the reference path's rule."""
    pro = PA.qkv_prologue_params(torch.zeros(1, 3 * D, dtype=o.dtype), 1, 1, D, out_scale=out_scale, **kw)
    return PA._out_quant_ref(o, pro)


def test_out_scale_int8_round_types_ties_and_bounds():
    # out_scale 1 / 127 with bound 127: a = 127 * fl(1/127) is exactly 1, so y = o
    o = torch.tensor([0.5, -0.5, 1.5, -1.5, 2.5, -2.5, 3.25, 200.0, -200.0, 126.5, -127.5, 0.0] + [0.0] * 4, dtype=torch.bfloat16)[None].repeat(1, 8)
    assert torch.tensor(127.0) * torch.tensor(1.0 / 127.0) == 1.0
    even = _out_quant(o, 1.0 / 127.0, quant_round_type=0, quant_max_bound=127.0, quant_min_bound=-127.0)
    away = _out_quant(o, 1.0 / 127.0, quant_round_type=1, quant_max_bound=127.0, quant_min_bound=-127.0)
    assert even.dtype == torch.int8 and away.dtype == torch.int8
    assert even[0, :12].tolist() == [0, 0, 2, -2, 2, -2, 3, 127, -127, 126, -127, 0]
    assert away[0, :12].tolist() == [1, -1, 2, -2, 3, -3, 3, 127, -127, 127, -127, 0]
    low = _out_quant(o, 1.0 / 127.0, quant_round_type=1, quant_max_bound=127.0, quant_min_bound=-100.0)
    assert low[0, 8].item() == -100


def test_out_scale_fp8_and_shift_smooth():
    g = torch.Generator().manual_seed(0)
    o = (torch.randn(4, 2 * D, generator=g) * 3).to(torch.float16)
    y = _out_quant(o, 0.01, quant_max_bound=448.0, quant_min_bound=-448.0)
    assert y.dtype == torch.float8_e4m3fn
    want = (torch.tensor(448.0) * torch.tensor(0.01) * o.float()).clamp(-448, 448).to(torch.float8_e4m3fn)
    assert torch.equal(y.view(torch.uint8), want.view(torch.uint8))
    shift = (torch.randn(2 * D, generator=g)).to(torch.float16)
    smooth = (torch.rand(2 * D, generator=g) + 0.5).to(torch.float16)
    pro = PA.qkv_prologue_params(torch.zeros(1, 4 * D, dtype=o.dtype), 2, 1, D, out_scale=0.02, out_shift=shift, out_smooth=smooth)
    y = PA._out_quant_ref(o, pro)
    z = torch.tensor(127.0) * torch.tensor(0.02) * ((o + shift) * smooth).float()
    assert torch.equal(y, PA._round_half_away(z).clamp(-127, 127).to(torch.int8))


def test_out_scale_through_the_op_and_ignored_shift_without_it():
    nh, nkv = 8, 2
    qkv, kc, vc, args, _ = mixed_batch(SPECS, nh, nkv, 16, torch.bfloat16, seed=4)
    plain = call(qkv.clone(), kc.clone(), vc.clone(), args)
    shift = torch.ones(nh * D, dtype=torch.bfloat16)
    assert torch.equal(call(qkv.clone(), kc.clone(), vc.clone(), args, out_shift=shift, out_smooth=shift)[0], plain[0])
    got = call(qkv.clone(), kc.clone(), vc.clone(), args, out_scale=0.05, quant_round_type=0)
    assert got[0].dtype == torch.int8
    assert torch.equal(got[0], _out_quant(plain[0], 0.05, quant_round_type=0))
    got = call(qkv.clone(), kc.clone(), vc.clone(), args, out_scale=0.05, quant_max_bound=448.0, quant_min_bound=-448.0)
    assert got[0].dtype == torch.float8_e4m3fn


def test_prologue_argument_errors():
    nh, nkv = 8, 2
    qkv, kc, vc, args, _ = mixed_batch(SPECS, nh, nkv, 16, torch.bfloat16, seed=5)
    w = qkv.shape[1]
    i32 = torch.zeros(qkv.shape, dtype=torch.int32)
    ones = torch.ones(w)
    cases = [
        (dict(qkv=i32, qkv_out_scale=ones), "compute_dtype"),                        # int32 with compute_dtype 'default'
        (dict(qkv=i32, compute_dtype="bf16"), "qkv_out_scale"),
        (dict(qkv=i32, qkv_out_scale=torch.ones(w - 1), compute_dtype="bf16"), "qkv_out_scale"),
        (dict(qkv_out_scale=ones), "int32"),                                         # qkv_out_scale with a float qkv
        (dict(compute_dtype="fp16"), "does not match"),
        (dict(compute_dtype="int8"), "compute_dtype"),
        (dict(rope_emb=torch.ones(2, 2, 128, 1, D // 2)), "batch dimension"),
        (dict(rope_emb=torch.ones(2, 1, 128, 1, D)), "last dimension"),
        (dict(rope_emb=torch.ones(2, 1, 128, 1, D // 2), use_neox_style=True), "last dimension"),
        (dict(rope_emb=torch.ones(3, 1, 128, 1, D // 2)), "rope_emb"),
        (dict(rope_emb=torch.ones(2, 1, 70, 1, D // 2)), "position 70"),            # the last decode row sits at position 70
        (dict(qkv_bias=torch.ones(w + 1, dtype=torch.bfloat16)), "qkv_bias"),
        (dict(out_scale=0.1, quant_max_bound=100.0, quant_min_bound=-100.0), "127"),
        (dict(out_scale=0.1, out_shift=torch.ones(nh * D, dtype=torch.bfloat16)), "together"),
        (dict(out_scale=0.1, out_smooth=torch.ones(nh * D, dtype=torch.bfloat16)), "together"),
        (dict(out_scale=0.1, out_shift=torch.ones(nh * D, dtype=torch.bfloat16), out_smooth=torch.ones(nh * D, dtype=torch.bfloat16),
              quant_max_bound=448.0, quant_min_bound=-448.0), "int8 output only"),
        (dict(out_scale=0.1, out_shift=torch.ones(3, dtype=torch.bfloat16), out_smooth=torch.ones(3, dtype=torch.bfloat16)), "H \\* D"),
    ]
    for kw, match in cases:
        x = kw.pop("qkv", qkv)
        k0, v0 = kc.clone(), vc.clone()
        with pytest.raises(ValueError, match=match):
            call(x.clone(), k0, v0, args, **kw)
        assert torch.equal(k0, kc) and torch.equal(v0, vc), kw                         # raised before anything was written
    call(qkv.clone(), kc.clone(), vc.clone(), args, rope_emb=torch.ones(2, 1, 71, 1, D // 2))   # position 70 is the table's last row


def test_no_prologue_input_is_the_old_call():
    qkv, kc, vc, args, _ = mixed_batch(SPECS, 8, 2, 16, torch.bfloat16, seed=6)
    assert PA.qkv_prologue_params(qkv, 8, 2, D, compute_dtype="bf16", out_scale=-1, use_neox_style=True) is None
    a = call(qkv.clone(), kc.clone(), vc.clone(), args)
    b = call(qkv.clone(), kc.clone(), vc.clone(), args, compute_dtype="bf16", use_neox_style=True, rope_theta=500000.0)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
