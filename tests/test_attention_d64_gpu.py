"""Training attention at head_dim 64 on the sm_90a kernels (csrc/attention_d64_sm100.cu), against two oracles:

1. The head_dim 128 kernels on the same operands zero-padded to 128 dims with the scale 1/sqrt(64) passed explicitly: the same
   function, computed by trusted kernels over the same 128-key tiles.  The first 64 columns of O, dK and dV, and dQ of the
   deterministic backward, must agree to one unit in the last place of the output dtype (lse: 4 fp32 ulps).
2. float64 attention on the kernels' own 16-bit inputs, element by element: |out - ref| <= 2 * bound, where bound sums the rounding
   the kernels are allowed and is computed from the magnitude of the terms:
   - the output's own rounding, u * |ref| (u = 2^-8 bf16, 2^-11 fp16: half an ulp of the dtype, doubled for the fp32 sums);
   - eta, half the smallest subnormal of the dtype (2^-25 in fp16), wherever a value is rounded to 16 bits: the outputs, and P and
     dS at every visible (query, key) pair, carried through the same sums as their relative rounding;
   - P rounded to 16 bits before P V and P^T dO: u * (|P| |V|) and u * (|P|^T |dO|);
   - dS rounded to 16 bits before dS^T Q and dS K, delta = rowsum(dO * O) taken on the 16-bit O, and dP = dO V^T summed in fp32:
     err(dS) = u |dS| + scale |P| (u rowsum(|dO| |O|) + 2^-16 |dO| |V|^T), so dK <= err(dS)^T |Q| and dQ <= err(dS) |K|;
   - lse: 1e-5 * (1 + |lse|) (fp32 sums and exp2 / log2 of 2^-22 relative error).
   A failure names the worst element and its bound.
"""
import math

import pytest
import torch
import torch.nn.functional as TF

import paddle_b200 as paddle
from paddle_b200 import kernels
from paddle_b200.kernels import attention as KAT

pytestmark = pytest.mark.gpu

SC = 64 ** -0.5
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
MANT = {torch.bfloat16: 7, torch.float16: 10}


def _ext():
    from paddle_b200._build import ext

    return ext()


def _deterministic(fn):
    paddle.set_flags({"FLAGS_cudnn_deterministic": True})
    try:
        return fn()
    finally:
        paddle.set_flags({"FLAGS_cudnn_deterministic": False})


def _inputs(b, sq, sk, h, hk, dtype, d=64, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda *s: (torch.randn(*s, device="cuda", generator=g) * 1.5).to(dtype)  # noqa: E731
    return mk(b, sq, h, d), mk(b, sk, hk, d), mk(b, sk, hk, d), mk(b, sq, h, d)


def _run(q, k, v, g, causal, colmask=None, det=False, scale=SC):
    """(out, lse, dq, dk, dv) of the own kernels, with the launch count of the backward."""
    E = _ext()
    out, lse = E.attention_fwd(q, k, v, scale, causal, False, colmask)
    kernels.reset_launch_count()
    fn = lambda: E.attention_bwd(q, k, v, out, lse, g, scale, causal, colmask)  # noqa: E731
    dq, dk, dv = _deterministic(fn) if det else fn()
    return (out, lse, dq, dk, dv), kernels.launch_count()


def _ulps(a, b, dtype):
    """|a - b| in units of the last place of dtype at |b| (b exact in dtype)."""
    a, b = a.double(), b.double()
    e = torch.floor(torch.log2(b.abs().clamp(min=torch.finfo(dtype).tiny)))
    return ((a - b).abs() / torch.exp2(e - MANT[dtype]))


def _check_padded(q, k, v, g, causal, colmask=None):
    """Oracle 1; returns the worst difference in ulps over O, dK, dV (one pass) and dQ (deterministic), and lse's absolute one."""
    dtype = q.dtype
    pad = lambda t: TF.pad(t, (0, 64)).contiguous()  # noqa: E731
    one, n1 = _run(q, k, v, g, causal, colmask)
    det, n2 = _run(q, k, v, g, causal, colmask, det=True)
    assert (n1, n2) == (2, 3), (n1, n2)
    ref, _ = _run(pad(q), pad(k), pad(v), pad(g), causal, colmask)
    ref_det, _ = _run(pad(q), pad(k), pad(v), pad(g), causal, colmask, det=True)
    worst = {}
    for name, a, r in (("out", one[0], ref[0]), ("dk", one[3], ref[3]), ("dv", one[4], ref[4]), ("dq", det[2], ref_det[2])):
        ul = _ulps(a, r[..., :64], dtype)
        worst[name] = ul.max().item() if ul.numel() else 0.0
        assert worst[name] <= 1.0, (name, worst[name], (ul == ul.max()).nonzero()[0].tolist())
    fin = torch.isfinite(ref[1])
    assert torch.equal(torch.isfinite(one[1]), fin)
    d = (one[1][fin] - ref[1][fin]).abs().max().item() if fin.any() else 0.0
    worst["lse"] = d
    assert d <= 4 * 2 ** -23 * max(1.0, ref[1][fin].abs().max().item() if fin.any() else 1.0), d
    return one, det, worst


def _ref64(q, k, v, g, causal, vis=None):
    """float64 O, lse, dQ, dK, dV and their rounding bounds (see the module docstring)."""
    u = U[q.dtype]
    b, sq, h, d = q.shape
    hk = k.shape[2]
    qd, kd, vd, gd = (t.double() for t in (q, k, v, g))
    kd, vd = kd.repeat_interleave(h // hk, 2), vd.repeat_interleave(h // hk, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", qd, kd) * SC
    sk = kd.shape[1]
    m = torch.ones(sq, sk, dtype=torch.bool, device=q.device)
    if causal:
        m = m.tril(sk - sq)
    m = m[None, None]
    if vis is not None:
        m = m & vis
    s = s.masked_fill(~m, float("-inf"))
    lse = torch.logsumexp(s, -1)                                               # [b, h, sq]
    p = torch.exp(s - lse.unsqueeze(-1)).nan_to_num(0.0)                       # fully masked rows: 0
    o = torch.einsum("bhqk,bkhd->bqhd", p, vd)
    dp = torch.einsum("bqhd,bkhd->bhqk", gd, vd)
    o16 = o.to(q.dtype).double()
    delta = (gd * o).sum(-1).transpose(1, 2)                                  # [b, h, sq]
    ds = p * (dp - delta.unsqueeze(-1)) * SC
    dq = torch.einsum("bhqk,bkhd->bqhd", ds, kd)
    dkf = torch.einsum("bhqk,bqhd->bkhd", ds, qd)
    dvf = torch.einsum("bhqk,bqhd->bkhd", p, gd)
    eta = torch.finfo(q.dtype).tiny * 2.0 ** -MANT[q.dtype] / 2               # half the smallest subnormal: the absolute rounding floor
    vis_f = m.expand_as(p).double()                                          # P and dS are rounded only where a key is visible
    e_ds = (u * ds.abs() + eta * vis_f + SC * p * u * (gd.abs() * o16.abs()).sum(-1).transpose(1, 2).unsqueeze(-1)
            + SC * p * 2.0 ** -16 * torch.einsum("bqhd,bkhd->bhqk", gd.abs(), vd.abs()))     # dP's fp32 sum over d
    bo = eta + u * o.abs() + torch.einsum("bhqk,bkhd->bqhd", u * p + eta * vis_f, vd.abs())
    bdq = eta + u * dq.abs() + torch.einsum("bhqk,bkhd->bqhd", e_ds, kd.abs())
    bdk = eta + u * dkf.abs() + torch.einsum("bhqk,bqhd->bkhd", e_ds, qd.abs())
    bdv = eta + u * dvf.abs() + torch.einsum("bhqk,bqhd->bkhd", u * p + eta * vis_f, gd.abs())
    fold = lambda t: t.reshape(b, sk, hk, h // hk, d).sum(3)  # noqa: E731   (query heads of a group add into one kv head)
    return (o, lse, dq, fold(dkf), fold(dvf)), (bo, None, bdq, fold(bdk), fold(bdv))


def _check_f64(res, q, k, v, g, causal, vis=None):
    ref, bnd = _ref64(q, k, v, g, causal, vis)
    worst = {}
    for name, a, r, bd in zip(("out", "lse", "dq", "dk", "dv"), res, ref, bnd):
        a = a.double()
        if name == "lse":
            fin = torch.isfinite(r)
            assert torch.equal(torch.isfinite(a), fin), "lse: -inf rows differ"
            a, r = a[fin], r[fin]
            bd = 1e-5 * (1 + r.abs())
        bd = 2 * bd
        err = (a - r).abs()
        if err.numel() == 0:
            continue
        frac = err / bd.clamp(min=1e-300)
        i = int(frac.argmax())
        worst[name] = frac.reshape(-1)[i].item()
        assert worst[name] <= 1.0, (name, "worst element", list(torch.unravel_index(torch.tensor(i), err.shape)) if err.dim() else i,
                                    "got", a.reshape(-1)[i].item(), "ref", r.reshape(-1)[i].item(), "bound", bd.reshape(-1)[i].item())
    return worst


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("h,hk", [(4, 4), (8, 2), (32, 4)])
@pytest.mark.parametrize("s", [1, 63, 64, 65, 127, 128, 129, 1000])
@pytest.mark.parametrize("b", [1, 3])
def test_d64_matches_padded_d128_and_float64(b, s, h, hk, causal, dtype):
    sk = s if causal else s + 37          # non-causal: sq != sk
    q, k, v, g = _inputs(b, s, sk, h, hk, dtype, seed=s + 7 * h)
    one, det, worst = _check_padded(q, k, v, g, causal)
    print(f"padded-D128 worst (ulps; lse abs) b={b} s={s} h={h}/{hk} causal={causal} {dtype}: {worst}")
    w1 = _check_f64(one, q, k, v, g, causal)
    w2 = _check_f64(det, q, k, v, g, causal)
    print(f"float64 worst fraction of bound: one-pass {w1} deterministic {w2}")


def test_d64_training_shape_matches_padded_d128():
    """TinyLlama's attention in training: B = 2, S = 2048, 32 / 4 heads."""
    q, k, v, g = _inputs(2, 2048, 2048, 32, 4, torch.bfloat16, seed=11)
    _, _, worst = _check_padded(q, k, v, g, True)
    print(f"training shape, padded-D128 worst: {worst}")


def test_d64_deterministic_is_bitwise_reproducible():
    q, k, v, g = _inputs(2, 777, 777, 8, 2, torch.bfloat16, seed=3)
    a, n = _run(q, k, v, g, True, det=True)
    c, _ = _run(q, k, v, g, True, det=True)
    assert n == 3
    for x, y in zip(a, c):
        assert torch.equal(x, y)


def _doc_colmask(b, s, cut):
    keys = torch.arange(s, device="cuda")
    se = torch.where(keys < cut, torch.full_like(keys, cut), torch.full_like(keys, s)).reshape(1, 1, s, 1).expand(b, 1, s, 1).int().contiguous()
    return se


def test_d64_fully_masked_row():
    """A query row hidden from every key: O = 0, lse = -inf, zero dQ, and nothing of it reaches dK / dV."""
    b, s, h = 2, 200, 4
    q, k, v, g = _inputs(b, s, s, h, 2, torch.bfloat16, seed=5)
    r0 = 77
    cm = torch.zeros(b, 1, s, 4, dtype=torch.int32, device="cuda")
    cm[..., 0], cm[..., 1] = r0, r0 + 1
    one, det, _ = _check_padded(q, k, v, g, False, cm)
    for res in (one, det):
        out, lse, dq = res[0], res[1], res[2]
        assert torch.all(out[:, r0] == 0) and torch.all(lse[:, :, r0] == float("-inf")) and torch.all(dq[:, r0] == 0)
        assert all(torch.isfinite(t).all() for t in (out, dq, res[3], res[4]))
    vis = KAT.colmask_to_dense(cm, s)
    print("fully masked row, float64:", _check_f64(one, q, k, v, g, False, vis))


@pytest.mark.parametrize("seq_major", [False, True])
def test_d64_packed_writes_dqkv_in_place(seq_major):
    """attention_packed at head_dim 64 runs the own kernels (launch count, no SDPA) and its d(qkv) equals the kernels' dq | dk | dv."""
    s, b, nh, nkv = 321, 2, 8, 2
    torch.manual_seed(5)
    shape = (s, b, nh + 2 * nkv, 64) if seq_major else (b, s, nh + 2 * nkv, 64)
    base = (torch.randn(*shape, device="cuda") * 0.7).to(torch.bfloat16)
    g = torch.randn(*shape[:2], nh, 64, device="cuda").to(torch.bfloat16)

    def grad():
        x = base.clone().requires_grad_(True)
        kernels.reset_launch_count()
        KAT.attention_packed(x, nh, nkv, True, None, seq_major=seq_major).backward(g)
        return x.grad, kernels.launch_count()

    xg, n = _deterministic(grad)
    assert n == 4, n                       # forward + stats + dK/dV + dQ: no copies, no slice gradients
    xb = base.transpose(0, 1) if seq_major else base
    gb = (g.transpose(0, 1) if seq_major else g).contiguous()
    res, _ = _run(xb[:, :, :nh].contiguous(), xb[:, :, nh:nh + nkv].contiguous(), xb[:, :, nh + nkv:].contiguous(), gb, True, det=True)
    xgb = xg.transpose(0, 1) if seq_major else xg
    for a, r in zip((xgb[:, :, :nh], xgb[:, :, nh:nh + nkv], xgb[:, :, nh + nkv:]), res[2:]):
        assert torch.equal(a, r.to(a.dtype))


@pytest.mark.parametrize("kind", ["flashmask_causal_doc", "flashmask_4", "varlen", "window"])
def test_d64_masked_variants_on_own_kernels(kind, monkeypatch):
    """flashmask / flash_attn_unpadded / flashmask_attention(window_size=...) at head_dim 64: no SDPA fallback, and forward and gradients
    match float64 under the same mask."""
    import paddle_b200.nn.functional as F

    def no_ref(*a, **kw):
        raise AssertionError("fell back to attention_ref")

    monkeypatch.setattr(KAT, "attention_ref", no_ref)
    B, S, H, D = 2, 384, 4, 64
    torch.manual_seed(3)
    mk = lambda *sh: (torch.randn(*sh, device="cuda") * 1.0).to(torch.bfloat16).requires_grad_(True)  # noqa: E731
    P = lambda t: t.as_subclass(paddle.Tensor)  # noqa: E731
    causal = False
    if kind == "varlen":
        cu = torch.tensor([0, 100, 280, 384], device="cuda", dtype=torch.int32)
        q, k, v = mk(S, H, D), mk(S, H, D), mk(S, H, D)
        causal = True
        kernels.reset_launch_count()
        out, _ = F.flash_attn_unpadded(P(q), P(k), P(v), cu, cu, 180, 180, SC, causal=True)
        vis = KAT.colmask_to_dense(KAT.colmask_from_cu_seqlens(cu, cu, S), S)
    else:
        q, k, v = mk(B, S, H, D), mk(B, S, H, D), mk(B, S, H, D)
        keys = torch.arange(S, device="cuda")
        kernels.reset_launch_count()
        if kind == "window":
            out = F.flashmask_attention(P(q), P(k), P(v), None, causal=False, window_size=(48, 16))
            vis = KAT.colmask_to_dense(KAT.colmask_from_window(S, S, 48, 16, False, q.device), S)
        else:
            if kind == "flashmask_causal_doc":
                causal = True
                se = _doc_colmask(B, S, 200)
            else:
                lts, lte = (keys + 64).clamp(max=S), (keys + 128).clamp(max=S)
                uts, ute = (keys - 160).clamp(min=0), (keys - 96).clamp(min=0)
                se = torch.stack([lts, lte, uts, ute], -1).reshape(1, 1, S, 4).expand(B, 1, S, 4).int().contiguous()
            out = F.flashmask_attention(P(q), P(k), P(v), se, causal=causal)
            vis = KAT.colmask_to_dense(KAT.colmask_from_startend(se, causal, S), S)
    assert kernels.launch_count() == 1, kernels.launch_count()
    out_t = out.as_subclass(torch.Tensor)
    g = torch.randn_like(out_t)
    kernels.reset_launch_count()
    out_t.backward(g)
    assert kernels.launch_count() == 2, kernels.launch_count()
    lift = (lambda t: t.unsqueeze(0)) if kind == "varlen" else (lambda t: t)
    qq, kk, vv, gg = (lift(t.detach()) for t in (q, k, v, g))
    ref, bnd = _ref64(qq, kk, vv, gg, causal, vis)
    for name, a, r, bd in (("out", lift(out_t), ref[0], bnd[0]), ("dq", lift(q.grad), ref[2], bnd[2]), ("dk", lift(k.grad), ref[3], bnd[3]),
                           ("dv", lift(v.grad), ref[4], bnd[4])):
        frac = ((a.double() - r).abs() / (2 * bd).clamp(min=1e-300)).max().item()
        assert frac <= 1.0, (kind, name, frac)


def _model_no_fallback(model_fn, cfg, monkeypatch, ids):
    def no_ref(*a, **kw):
        raise AssertionError("fell back to attention_ref")

    monkeypatch.setattr(KAT, "attention_ref", no_ref)
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        model = model_fn(cfg)
        loss = model(ids[:, :-1], ids[:, 1:])
        loss.backward()
        assert math.isfinite(float(loss.item()))
        assert all(p.grad is not None and bool(torch.isfinite(p.grad.as_subclass(torch.Tensor)).all()) for p in model.parameters() if not p.stop_gradient)
    finally:
        paddle.set_default_dtype("float32")


@pytest.mark.parametrize("window", [None, 100])
def test_d64_llama_runs_on_own_kernels(window, monkeypatch):
    from paddle_b200.models import LlamaForCausalLM, llama_tiny

    paddle.set_device("gpu:0")
    cfg = llama_tiny(hidden_size=256, num_attention_heads=4, num_key_value_heads=2, intermediate_size=512, vocab_size=1024,
                     max_position_embeddings=512, sliding_window=window)
    assert cfg.head_dim == 64
    _model_no_fallback(LlamaForCausalLM, cfg, monkeypatch, paddle.randint(0, cfg.vocab_size, [2, 301]))


def test_d64_gpt_runs_on_own_kernels(monkeypatch):
    from paddle_b200.models import GPTForCausalLM, gpt_tiny

    paddle.set_device("gpu:0")
    cfg = gpt_tiny(hidden_size=256, num_attention_heads=4, intermediate_size=1024, vocab_size=1024, max_position_embeddings=512)
    _model_no_fallback(GPTForCausalLM, cfg, monkeypatch, paddle.randint(0, cfg.vocab_size, [2, 301]))


def test_tinyllama_two_layers_match_sdpa():
    """tinyllama_1b() cut to 2 layers, bf16: loss within 2e-3 relative and every parameter gradient within 3e-2 relative norm of the
    same model on torch SDPA (FLAGS_b200_flash_attention=0).  Both arms round P, dS and the activations to bf16 in different places;
    the bounds are about ten bf16 ulps on the loss and a few percent on gradient norms, the spread of two valid bf16 attentions."""
    from paddle_b200.models import LlamaForCausalLM, tinyllama_1b

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        cfg = tinyllama_1b(num_hidden_layers=2)
        paddle.seed(0)
        model = LlamaForCausalLM(cfg)
        ids = paddle.randint(0, cfg.vocab_size, [2, 1025])

        def step():
            model.clear_gradients()
            kernels.reset_launch_count()
            loss = model(ids[:, :-1], ids[:, 1:])
            loss.backward()
            return float(loss.item()), {n: p.grad.as_subclass(torch.Tensor).float().clone() for n, p in model.named_parameters()}

        own = step()
        paddle.set_flags({"FLAGS_b200_flash_attention": False})
        try:
            sdpa = step()
        finally:
            paddle.set_flags({"FLAGS_b200_flash_attention": True})
    finally:
        paddle.set_default_dtype("float32")
    assert abs(own[0] - sdpa[0]) <= 2e-3 * abs(sdpa[0]), (own[0], sdpa[0])
    worst = max(((own[1][n] - sdpa[1][n]).norm() / sdpa[1][n].norm().clamp(min=1e-12)).item() for n in sdpa[1])
    print(f"tinyllama 2 layers: loss own {own[0]:.6f} sdpa {sdpa[0]:.6f}, worst gradient relative norm difference {worst:.4f}")
    for n in sdpa[1]:
        r = ((own[1][n] - sdpa[1][n]).norm() / sdpa[1][n].norm().clamp(min=1e-12)).item()
        assert r < 3e-2, (n, r)
