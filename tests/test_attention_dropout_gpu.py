"""Attention dropout on the sm_90a flash-attention kernels (csrc/attention_dropout_sm100.cu), against kernels.attention.dropout_keep_mask:

1. Exact mask readout: with q = k = 0 every visible key has P = 1 / n_visible, and with V[j] = e_j the output is
   O[b, i, h, j] = Z[b, h, i, j] / ((1 - p) n_visible), so its zero pattern is the mask itself.
2. float64 attention with the reference mask of the seed_offset the forward returned, element by element, under the rounding bound of
   tests/test_attention_d64_gpu.py with P replaced by the dropped and rescaled Zs P = Z P / (1 - p) wherever it is rounded or summed.
3. Head_dim 64 against the head_dim 128 kernels on zero-padded operands with the same fixed seed_offset: the mask does not depend on D.
4. Reproducibility and the generator; 5. unchanged routing at p = 0 / eval / p >= 1; 6. CUDA graphs; 7. a GPT with attention dropout.
"""
import math

import pytest
import torch
import torch.nn.functional as TF

import paddle_b200 as paddle
from paddle_b200 import kernels
from paddle_b200.kernels import attention as KAT
from paddle_b200.kernels.attention import dropout_keep_mask

pytestmark = pytest.mark.gpu

U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
MANT = {torch.bfloat16: 7, torch.float16: 10}
P = 0.1


def _ext():
    from paddle_b200._build import ext

    return ext()


def _deterministic(fn):
    paddle.set_flags({"FLAGS_cudnn_deterministic": True})
    try:
        return fn()
    finally:
        paddle.set_flags({"FLAGS_cudnn_deterministic": False})


def _inputs(b, sq, sk, h, hk, dtype, d, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda *s: (torch.randn(*s, device="cuda", generator=g) * 1.5).to(dtype)  # noqa: E731
    return mk(b, sq, h, d), mk(b, sk, hk, d), mk(b, sk, hk, d), mk(b, sq, h, d)


def _mask(so, b, h, sq, sk, p=P):
    s, o = (int(x) for x in so.cpu())
    return dropout_keep_mask(s, o, b, h, sq, sk, p, device="cuda")


def _vis(sq, sk, causal, colmask=None, device="cuda"):
    m = torch.ones(sq, sk, dtype=torch.bool, device=device)
    if causal:
        m = m.tril(sk - sq)
    m = m[None, None]
    if colmask is not None:
        m = m & KAT.colmask_to_dense(colmask, sq)
    return m


# ---------------------------------------------------------------------------------------------------- 1. exact mask readout
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("causal,sq,sk", [(False, 77, 61), (True, 61, 61), (False, 130, 64)])
@pytest.mark.parametrize("masked", [False, True])
def test_mask_readout(dtype, d, causal, sq, sk, masked):
    b, h, hk = 2, 4, 2
    q = torch.zeros(b, sq, h, d, dtype=dtype, device="cuda")
    k = torch.zeros(b, sk, hk, d, dtype=dtype, device="cuda")
    v = torch.zeros(b, sk, hk, d, dtype=dtype, device="cuda")
    v[:, torch.arange(sk), :, torch.arange(sk)] = 1                     # V[j] = e_j
    cm = KAT.colmask_from_window(sq, sk, 20, 9, causal, "cuda").expand(b, -1, -1, -1).contiguous() if masked else None
    out, lse, so = _ext().attention_fwd(q, k, v, 0.125, causal, False, cm, P, None)
    vis = _vis(sq, sk, causal, cm).expand(b, h, sq, sk)
    z = _mask(so, b, h, sq, sk)
    o = out[..., :sk].permute(0, 2, 1, 3)                               # [b, h, sq, sk]
    assert torch.equal(o != 0, z & vis)
    n = vis.sum(-1, keepdim=True).clamp(min=1).double()
    ref = (z & vis).double() / ((1 - P) * n)
    assert ((o.double() - ref).abs() <= U[dtype] * ref + 1e-30).all()


# ---------------------------------------------------------------------------------------------------- 2. float64 with the mask
def _ref64(q, k, v, g, causal, z, sc, vis=None, p=P):
    u = U[q.dtype]
    b, sq, h, d = q.shape
    hk = k.shape[2]
    qd, kd, vd, gd = (t.double() for t in (q, k, v, g))
    kd, vd = kd.repeat_interleave(h // hk, 2), vd.repeat_interleave(h // hk, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", qd, kd) * sc
    sk = kd.shape[1]
    m = _vis(sq, sk, causal)
    if vis is not None:
        m = m & vis
    s = s.masked_fill(~m, float("-inf"))
    lse = torch.logsumexp(s, -1)
    pr = torch.exp(s - lse.unsqueeze(-1)).nan_to_num(0.0)
    zs = z.double() / (1 - p)
    pz = pr * zs
    o = torch.einsum("bhqk,bkhd->bqhd", pz, vd)
    dp = torch.einsum("bqhd,bkhd->bhqk", gd, vd)
    o16 = o.to(q.dtype).double()
    delta = (gd * o).sum(-1).transpose(1, 2)
    ds = pr * (zs * dp - delta.unsqueeze(-1)) * sc
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kd)
    dkf = torch.einsum("bhqk,bqhd->bkhd", ds, qd)
    dvf = torch.einsum("bhqk,bqhd->bkhd", pz, gd)
    eta = torch.finfo(q.dtype).tiny * 2.0 ** -MANT[q.dtype] / 2
    vis_f = m.expand_as(pr).double()
    e_ds = (u * ds.abs() + eta * vis_f + sc * pr * u * (gd.abs() * o16.abs()).sum(-1).transpose(1, 2).unsqueeze(-1)
            + sc * pz * 2.0 ** -16 * torch.einsum("bqhd,bkhd->bhqk", gd.abs(), vd.abs()))
    bo = eta + u * o.abs() + torch.einsum("bhqk,bkhd->bqhd", u * pz + eta * vis_f, vd.abs())
    bdq = eta + u * dq.abs() + torch.einsum("bhqk,bkhd->bqhd", e_ds, kd.abs())
    bdk = eta + u * dkf.abs() + torch.einsum("bhqk,bqhd->bkhd", e_ds, qd.abs())
    bdv = eta + u * dvf.abs() + torch.einsum("bhqk,bqhd->bkhd", u * pz + eta * vis_f, gd.abs())
    fold = lambda t: t.reshape(b, sk, hk, h // hk, d).sum(3)  # noqa: E731
    return (o, lse, dq, fold(dkf), fold(dvf)), (bo, None, bdq, fold(bdk), fold(bdv))


WORST = {}


def _check_f64(tag, res, q, k, v, g, causal, so, sc, vis=None):
    b, sq, h, _ = q.shape
    z = _mask(so, b, h, sq, k.shape[1])
    ref, bnd = _ref64(q, k, v, g, causal, z, sc, vis)
    for name, a, r, bd in zip(("out", "lse", "dq", "dk", "dv"), res, ref, bnd):
        if a is None:
            continue
        a = a.double()
        if name == "lse":
            fin = torch.isfinite(r)
            assert torch.equal(torch.isfinite(a), fin)
            a, r = a[fin], r[fin]
            bd = 1e-5 * (1 + r.abs())
        bd = 2 * bd
        err = (a - r).abs()
        if err.numel() == 0:
            continue
        frac = err / bd.clamp(min=1e-300)
        i = int(frac.argmax())
        w = frac.reshape(-1)[i].item()
        WORST[name] = max(WORST.get(name, 0.0), w)
        assert w <= 1.0, (tag, name, "worst element", i, "got", a.reshape(-1)[i].item(), "ref", r.reshape(-1)[i].item(), "bound", bd.reshape(-1)[i].item())


SHAPES = [(2, 200, 200, 4, 2, True), (2, 200, 200, 4, 4, False), (1, 97, 301, 4, 1, False), (1, 256, 256, 2, 2, True)]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(str(int(x)) for x in s))
@pytest.mark.parametrize("det", [False, True])
def test_dense_against_float64(dtype, d, shape, det):
    b, sq, sk, h, hk, causal = shape
    q, k, v, g = _inputs(b, sq, sk, h, hk, dtype, d)
    sc = d ** -0.5
    E = _ext()
    out, lse, so = E.attention_fwd(q, k, v, sc, causal, False, None, P, None)
    kernels.reset_launch_count()
    fn = lambda: E.attention_bwd(q, k, v, out, lse, g, sc, causal, None, P, so)  # noqa: E731
    dq, dk, dv = _deterministic(fn) if det else fn()
    assert kernels.launch_count() == (3 if det else 2)
    _check_f64("dense", (out, lse, dq, dk, dv), q, k, v, g, causal, so, sc)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("front", ["flashmask", "varlen", "window"])
def test_colmask_front_ends_against_float64(dtype, d, front):
    from paddle_b200.nn import functional as F

    b, s, h, hk = 2, 300, 4, 2
    q, k, v, g = _inputs(b, s, s, h, hk, dtype, d, seed=3)
    fixed = torch.tensor([1234, 5678], dtype=torch.int64)
    sc = d ** -0.5
    if front == "varlen":
        cu = torch.tensor([0, 100, 251, 300, 450, 600], dtype=torch.int32, device="cuda")
        qf, kf, vf, gf = (t.reshape(b * s, t.shape[2], d) for t in (q, k, v, g))
        qs, ks, vs = (t.detach().clone().requires_grad_(True) for t in (qf, kf, vf))
        out, _ = F.flash_attn_unpadded(qs, ks, vs, cu, cu, 300, 300, sc, dropout=P, causal=True, fixed_seed_offset=fixed)
        torch.autograd.backward(out, gf)
        cm = KAT.colmask_from_cu_seqlens(cu, cu, b * s)
        one = lambda t: t.reshape(1, b * s, -1, d)  # noqa: E731
        vis = KAT.colmask_to_dense(cm, b * s)
        res = (one(out), None, one(qs.grad), one(ks.grad), one(vs.grad))
        _check_f64(front, res, one(qf), one(kf), one(vf), one(gf), True, fixed, sc, vis)
        return
    qs, ks, vs = (t.detach().clone().requires_grad_(True) for t in (q, k, v))
    if front == "flashmask":
        idx = torch.tensor([s] * 100 + [200] * 100 + [s] * 100, dtype=torch.int32, device="cuda").reshape(1, 1, s, 1).expand(b, 1, s, 1)
        out, so = F.flashmask_attention(qs, ks, vs, idx.contiguous(), dropout=P, causal=True, return_seed_offset=True)
        cm = KAT.colmask_from_startend(idx, True, s)
    else:
        out, so = F.flashmask_attention(qs, ks, vs, None, dropout=P, causal=True, window_size=64, return_seed_offset=True)
        cm = KAT.colmask_from_window(s, s, 64, 64, True, "cuda")
    torch.autograd.backward(out, g)
    out = out.as_subclass(torch.Tensor)
    res = (out, None, qs.grad, ks.grad, vs.grad)
    _check_f64(front, res, q, k, v, g, True, so, sc, KAT.colmask_to_dense(cm, s))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("seq_major", [False, True])
def test_packed_against_float64(dtype, d, seq_major):
    b, s, nh, nkv = 2, 190, 4, 2
    g0 = torch.Generator(device="cuda").manual_seed(5)
    shape = (s, b, nh + 2 * nkv, d) if seq_major else (b, s, nh + 2 * nkv, d)
    qkv = (torch.randn(*shape, device="cuda", generator=g0) * 1.5).to(dtype).requires_grad_(True)
    out, so = KAT.attention_packed(qkv, nh, nkv, causal=True, seq_major=seq_major, dropout_p=P, return_seed_offset=True)
    go = (torch.randn(*out.shape, device="cuda", generator=g0) * 1.5).to(dtype)
    torch.autograd.backward(out, go)
    x = qkv.detach().transpose(0, 1) if seq_major else qkv.detach()
    dx = qkv.grad.transpose(0, 1) if seq_major else qkv.grad
    bs = (lambda t: t.transpose(0, 1)) if seq_major else (lambda t: t)
    q, k, v = x[:, :, :nh], x[:, :, nh:nh + nkv], x[:, :, nh + nkv:]
    res = (bs(out.as_subclass(torch.Tensor)), None, dx[:, :, :nh], dx[:, :, nh:nh + nkv], dx[:, :, nh + nkv:])
    _check_f64("packed", res, q, k, v, bs(go), True, so, d ** -0.5)


# ---------------------------------------------------------------------------------------------------- 3. D 64 = padded D 128
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("causal", [False, True])
def test_d64_equals_padded_d128(dtype, causal):
    b, s, h, hk = 2, 333, 4, 2
    q, k, v, g = _inputs(b, s, s, h, hk, dtype, 64, seed=9)
    fixed = torch.tensor([99, 12345], dtype=torch.int64, device="cuda")
    E = _ext()
    pad = lambda t: TF.pad(t, (0, 64)).contiguous()  # noqa: E731

    def run(q, k, v, g, det):
        out, lse, so = E.attention_fwd(q, k, v, 0.125, causal, False, None, P, fixed)
        fn = lambda: E.attention_bwd(q, k, v, out, lse, g, 0.125, causal, None, P, so)  # noqa: E731
        return (out,) + tuple(_deterministic(fn) if det else fn())

    a, r = run(q, k, v, g, False), run(pad(q), pad(k), pad(v), pad(g), False)
    ad, rd = run(q, k, v, g, True), run(pad(q), pad(k), pad(v), pad(g), True)
    for name, x, y in (("out", a[0], r[0]), ("dk", a[2], r[2]), ("dv", a[3], r[3]), ("dq", ad[1], rd[1])):
        y = y[..., :64]
        e = torch.floor(torch.log2(y.double().abs().clamp(min=torch.finfo(dtype).tiny)))
        ul = ((x.double() - y.double()).abs() / torch.exp2(e - MANT[dtype])).max().item()
        assert ul <= 1.0, (name, ul)


# ---------------------------------------------------------------------------------------------------- 4. reproducibility
def test_reproducibility_and_generator():
    from paddle_b200.nn import functional as F

    q, k, v, g = _inputs(2, 256, 256, 4, 4, torch.bfloat16, 64, seed=1)
    E = _ext()
    fixed = torch.tensor([7, 4000], dtype=torch.int64)
    a = E.attention_fwd(q, k, v, 0.125, True, False, None, P, fixed)
    b = E.attention_fwd(q, k, v, 0.125, True, False, None, P, fixed)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2].cpu(), fixed)
    grads = [_deterministic(lambda: E.attention_bwd(q, k, v, a[0], a[1], g, 0.125, True, None, P, a[2])) for _ in range(2)]
    assert all(torch.equal(x, y) for x, y in zip(*grads))
    c = E.attention_fwd(q, k, v, 0.125, True, False, None, P, None)
    d = E.attention_fwd(q, k, v, 0.125, True, False, None, P, None)
    assert not torch.equal(c[2], d[2]) and not torch.equal(c[0], d[0])
    assert d[2][1].item() - c[2][1].item() >= 2 * 4                    # each call reserves B*H generator offsets
    paddle.seed(31)
    e1 = [E.attention_fwd(q, k, v, 0.125, True, False, None, P, None) for _ in range(2)]
    paddle.seed(31)
    e2 = [E.attention_fwd(q, k, v, 0.125, True, False, None, P, None) for _ in range(2)]
    for x, y in zip(e1, e2):
        assert torch.equal(x[0], y[0]) and torch.equal(x[2], y[2])
    idx = torch.full((2, 1, 256, 1), 256, dtype=torch.int32, device="cuda")
    out, so = F.flashmask_attention(q, k, v, idx, dropout=P, causal=True, return_seed_offset=True)
    again = F.flashmask_attention(q, k, v, idx, dropout=P, causal=True, fixed_seed_offset=so)
    assert torch.equal(out.as_subclass(torch.Tensor), again.as_subclass(torch.Tensor))


# ---------------------------------------------------------------------------------------------------- 5. routing
def test_routing_unchanged_without_dropout():
    from paddle_b200.nn import functional as F

    q, k, v, g = _inputs(2, 200, 200, 4, 2, torch.bfloat16, 128, seed=2)
    E = _ext()
    ref_out, ref_lse = E.attention_fwd(q, k, v, 128 ** -0.5, True)
    for fn in (lambda: F.flash_attention(q, k, v, dropout=0.0, causal=True)[0],
               lambda: F.flash_attention(q, k, v, dropout=0.3, causal=True, training=False)[0],
               lambda: F.scaled_dot_product_attention(q, k, v, None, 0.3, True, training=False)):
        kernels.reset_launch_count()
        out = fn()
        assert kernels.launch_count() == 1
        assert torch.equal(out.as_subclass(torch.Tensor), ref_out)
    qs = q.detach().clone().requires_grad_(True)
    out = KAT.attention(qs, k, v, None, 0.0, True)
    kernels.reset_launch_count()
    out.backward(g)
    assert kernels.launch_count() == 2
    assert torch.equal(qs.grad, E.attention_bwd(q, k, v, ref_out, ref_lse, g, 128 ** -0.5, True)[0])
    assert not KAT.fused_ok(q, k, v, None, 1.0, True)                  # dropout >= 1 and dense masks: SDPA
    assert not KAT.fused_ok(q, k, v, torch.ones(200, 200, dtype=torch.bool, device="cuda"), 0.1, False)
    assert KAT.fused_ok(q, k, v, None, 0.1, True)


# ---------------------------------------------------------------------------------------------------- 6. CUDA graphs and 7. model
def _gpt(attention_dropout, layers=2):
    from paddle_b200.models import GPTForCausalLM, gpt_tiny

    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = gpt_tiny(hidden_size=256, num_attention_heads=4, num_hidden_layers=layers, vocab_size=512, max_position_embeddings=256,
                       attention_dropout=attention_dropout)
        return GPTForCausalLM(cfg)
    finally:
        paddle.set_default_dtype("float32")


class _Record:
    """Wraps KAT.attention: records (q, k, v, out, seed_offset) of every dropout call; with `replay`, computes attention in float32 on the
    recorded masks instead."""

    def __init__(self, replay=None, capturing_only=False):
        self.calls, self.replay, self.orig, self.capturing_only = [], replay, KAT.attention, capturing_only

    def __call__(self, q, k, v, mask=None, dropout_p=0.0, causal=False, scale=None, **kw):
        if self.replay is not None:
            so = self.replay.pop(0)
            qr, kr, vr = (t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) else t for t in (q, k, v))
            b, s, h, d = qr.shape
            z = _mask(so, b, h, s, kr.shape[1], dropout_p).float() / (1 - dropout_p)
            sc = torch.einsum("bqhd,bkhd->bhqk", qr.float(), kr.float()) * d ** -0.5
            sc = sc.masked_fill(~_vis(s, kr.shape[1], causal), float("-inf"))
            pr = torch.softmax(sc, -1) * z
            return KAT.wrap(torch.einsum("bhqk,bkhd->bqhd", pr, vr.float()).to(qr.dtype))
        out, so = self.orig(q, k, v, mask, dropout_p, causal, scale, return_seed_offset=True)
        if not self.capturing_only or torch.cuda.is_current_stream_capturing():
            self.calls.append((q, k, v, out, so))
        return out


def test_gpt_trains_on_dropout_kernels(monkeypatch):
    monkeypatch.setattr(KAT, "attention_ref", lambda *a, **k: (_ for _ in ()).throw(AssertionError("attention_ref reached")))
    model = _gpt(0.1)
    model.train()
    ids = torch.randint(0, 512, (2, 129), device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
    rec = _Record()
    monkeypatch.setattr(KAT, "attention", rec)
    loss = model(ids[:, :-1], ids[:, 1:])
    loss.backward()
    assert len(rec.calls) == 2 and all(c[4] is not None for c in rec.calls)
    sos = [c[4].clone() for c in rec.calls]
    monkeypatch.setattr(KAT, "attention", _Record(replay=list(sos)))
    with torch.no_grad():
        ref = model(ids[:, :-1], ids[:, 1:])
    a, r = float(loss), float(ref)
    assert math.isfinite(a) and abs(a - r) <= 2e-3 * abs(r), (a, r)


def test_captured_train_step_draws_fresh_masks(monkeypatch):
    model = _gpt(0.1, layers=1)
    model.train()
    opt = paddle.optimizer.AdamW(1e-4, parameters=model.parameters(), multi_precision=True)
    opt.enable_flat_arena()
    ids = torch.randint(0, 512, (2, 65), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    rec = _Record(capturing_only=True)      # the graph's own tensors: every replay rewrites them
    monkeypatch.setattr(KAT, "attention", rec)
    step = paddle.jit.capture_train_step(lambda x, y: model(x, y), opt, warmup=1)
    pairs = []
    for i in range(4):
        loss = float(step(ids[:, :-1], ids[:, 1:]))
        assert math.isfinite(loss)
        if i < 2:                           # eager warm-up, then the recording (which returns the side-stream step's loss)
            continue
        assert step.captured, step.failure_traceback
        q, k, v, out, so = rec.calls[-1]
        pairs.append(so.clone())
        # this replay's output is the attention of the mask of the pair it recorded
        qr, kr, vr = (t.as_subclass(torch.Tensor) for t in (q, k, v))
        b, s, h, d = qr.shape
        z = _mask(so, b, h, s, s).double() / (1 - P)
        sc = torch.einsum("bqhd,bkhd->bhqk", qr.double(), kr.double()) * d ** -0.5
        pr = torch.softmax(sc.masked_fill(~_vis(s, s, True), float("-inf")), -1) * z
        ref = torch.einsum("bhqk,bkhd->bqhd", pr, vr.double())
        got = out.as_subclass(torch.Tensor).double()
        assert (got - ref).abs().max().item() <= 0.02 * ref.abs().max().item()
    assert step.replays == 2
    assert not torch.equal(pairs[0], pairs[1])                        # two replays, two masks
