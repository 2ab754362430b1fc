"""The kernels every training step runs (csrc/norm.cu, loss.cu, elementwise.cu, optim.cu) against float64 references.

Each reference is plain torch in float64 on the kernel's actual inputs (the bf16 / fp16 values the kernel reads), and
outputs are compared element by element: |out - ref| <= atol + rtol * |ref|.  rtol is about two rounding steps of the
output dtype.  Where the fp32 arithmetic inside a kernel cancels (a difference of large terms, a long sum), atol is
K_SUM fp32 rounding steps of the magnitude of the terms, computed from the same float64 inputs.  Shapes are picked so
that every launch path runs: each (threads, vectors-per-thread) shape of the norm kernels, persistent backward grids
with several rows per CTA and a partial last lap, vector and scalar-tail rows of the loss kernels, aligned and
unaligned optimizer slabs.  A failing check names the worst element."""
import math

import pytest
import torch
import torch.nn.functional as F

from paddle_b200 import kernels
from paddle_b200.kernels import activation as KA
from paddle_b200.kernels import loss as KL
from paddle_b200.kernels import norm as KN
from paddle_b200.kernels import rope as KR

pytestmark = pytest.mark.gpu

BF16, FP16, FP32 = torch.bfloat16, torch.float16, torch.float32
U32 = 2.0 ** -24                                        # fp32 unit roundoff
K_SUM = 64                                              # fp32 rounding steps allowed on the magnitude of the summed terms
RTOL = {BF16: 2.0 ** -7, FP16: 2.0 ** -10, FP32: 4e-6}  # ~2 ulp of the output dtype; fp32: rsqrtf / __expf / fp32 sums


def _ext():
    from paddle_b200._build import ext

    return ext()


def _t(x):
    return x.as_subclass(torch.Tensor) if isinstance(x, torch.Tensor) else x


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _lap_rows():
    """Rows for the persistent norm backward (grid = 4 * SMs CTAs): two full laps per CTA and a partial third."""
    return 2 * 4 * _sms() + 37


def check(what, out, ref, rtol, atol=0.0):
    """Element-wise |out - ref| <= atol + rtol * |ref| (atol may be a tensor); names the worst element on failure."""
    out = _t(out).detach()
    ref = ref.detach().to(torch.float64)
    assert out.shape == ref.shape, (what, tuple(out.shape), tuple(ref.shape))
    sub = torch.finfo(out.dtype).tiny * torch.finfo(out.dtype).eps  # spacing of the output dtype's subnormals
    o = out.to(torch.float64)
    err = (o - ref).abs()
    bound = atol + rtol * ref.abs() + sub
    ratio = torch.where(err <= bound, err / bound, torch.full_like(err, math.inf))  # NaN out -> inf
    worst = int(ratio.reshape(-1).argmax())
    idx = tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), ratio.shape)) if ratio.dim() else ()
    w_out, w_ref = o.reshape(-1)[worst].item(), ref.reshape(-1)[worst].item()
    rel = err.reshape(-1)[worst].item() / max(abs(w_ref), 1e-300)
    print(f"[tol] {what}: worst err/bound {ratio.reshape(-1)[worst].item():.3g} at {idx} "
          f"(out {w_out:.6g}, ref {w_ref:.6g}, rel {rel:.3g}, rtol {rtol:.3g})")
    bad = int((ratio == math.inf).sum())
    assert bad == 0, (f"{what}: {bad} of {ratio.numel()} elements outside atol + rtol*|ref| (rtol {rtol:.3g}); worst at {idx}: "
                      f"out {w_out!r}, ref {w_ref!r}, bound {bound.reshape(-1)[worst].item():.3g}")


def launches(fn):
    n0 = kernels.launch_count()
    out = fn()
    assert kernels.launch_count() > n0, "the op did not reach the native kernel"
    return out


# ------------------------------------------------------------------------------------------------ RMSNorm / LayerNorm
# cols per dtype: every (threads, VPT) branch of pick_shape, forward and backward; 11008 and 16384 are VPT 8 for 16-bit types
_COLS16 = [64, 1000, 2056, 5120, 11008, 16384]
NORM_SHAPES = [(BF16, c) for c in _COLS16] + [(FP16, c) for c in _COLS16] + [(FP32, c) for c in (512, 2056, 8192)]
NORM_ROWS = ["1", "300", "laps"]


def _rows(r):
    return _lap_rows() if r == "laps" else int(r)


def _norm_ref(kind, x, w, b, eps):
    """float64 RMSNorm / LayerNorm, plus the per-element magnitude of the terms the kernel sums in fp32."""
    if kind == "rms":
        r = torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps)
        xh, mag = x * r, None
    else:
        mu = x.mean(-1, keepdim=True)
        r = torch.rsqrt((x - mu).pow(2).mean(-1, keepdim=True) + eps)
        xh, mag = (x - mu) * r, r * x.abs().mean(-1, keepdim=True)   # error of the fp32 mean, carried into x_hat
    y = xh * w if w is not None else xh
    return (y + b if b is not None else y), r, xh, mag


def _run_norm(kind, dtype, rows, cols, affine=True, offset=0.0, seed=0):
    torch.manual_seed(seed)
    x = (torch.randn(rows, cols, device="cuda") + offset).to(dtype).requires_grad_(True)
    w = (torch.rand(cols, device="cuda") + 0.5).to(dtype).requires_grad_(True) if affine else None
    b = (torch.randn(cols, device="cuda")).to(dtype).requires_grad_(True) if affine and kind == "ln" else None
    eps = 1e-6 if kind == "rms" else 1e-5
    y = launches(lambda: _t(KN.rms_norm(x, w, eps)) if kind == "rms" else _t(KN.layer_norm(x, [cols], w, b, eps)))
    dy = torch.randn_like(y)
    y.backward(dy)

    x64, w64, b64 = (t.detach().double().requires_grad_(True) if t is not None else None for t in (x, w, b))
    y64, r, xh, mag = _norm_ref(kind, x64, w64, b64, eps)
    y64.backward(dy.double())
    g = dy.double()
    xh, r = xh.detach(), r.detach()
    wv = w64.detach() if w is not None else torch.ones(cols, device="cuda", dtype=torch.float64)
    gw = g * wv
    rt = RTOL[dtype]
    tag = f"{kind} {str(dtype)[6:]} {rows}x{cols}"

    y_mag = xh.abs() * wv.abs() + (b64.detach().abs() if b is not None else 0.0)
    if mag is not None:
        y_mag = y_mag + mag * wv.abs()
    check(f"{tag} y", y, y64, rt, K_SUM * U32 * y_mag)
    dx_mag = r * (gw.abs() + xh.abs() * (gw * xh).abs().mean(-1, keepdim=True))
    if kind == "ln":
        # the fp32 mean's error moves x_hat by mag; dx = r (gw - mean(gw) - x_hat mean(gw x_hat)) carries it twice
        dx_mag = (dx_mag + r * gw.abs().mean(-1, keepdim=True)
                  + r * mag * ((gw * xh).abs().mean(-1, keepdim=True) + xh.abs() * gw.abs().mean(-1, keepdim=True)))
    check(f"{tag} dx", x.grad, x64.grad, rt, K_SUM * U32 * dx_mag)
    if w is not None:
        dw_mag = (g.abs() * (xh.abs() + (mag if mag is not None else 0.0))).sum(0)
        check(f"{tag} dw", w.grad, w64.grad, rt, K_SUM * U32 * dw_mag)
    else:
        assert x.grad is not None
    if b is not None:
        check(f"{tag} db", b.grad, b64.grad, rt, K_SUM * U32 * g.abs().sum(0))


@pytest.mark.parametrize("rows", NORM_ROWS)
@pytest.mark.parametrize("dtype,cols", NORM_SHAPES)
@pytest.mark.parametrize("kind", ["rms", "ln"])
def test_norm_fwd_bwd_elementwise(kind, dtype, cols, rows):
    _run_norm(kind, dtype, _rows(rows), cols)


@pytest.mark.parametrize("dtype,cols", [(BF16, 1000), (FP16, 11008), (FP32, 2056)])
@pytest.mark.parametrize("kind", ["rms", "ln"])
def test_norm_without_weight(kind, dtype, cols):
    """rms_norm(x, None) and layer_norm(x, None, None): the kernels run with null w / b pointers."""
    _run_norm(kind, dtype, _lap_rows(), cols, affine=False, seed=1)


@pytest.mark.parametrize("cols", [2056, 8192])
def test_layer_norm_fp32_large_mean(cols):
    """x = 1e3 + randn: a one-pass variance (E[x^2] - E[x]^2) loses the unit variance to cancellation; the two-pass
    kernel keeps every element within the fp32 error of the mean (atol ~ K_SUM * 2^-24 * 1e3 * rstd)."""
    _run_norm("ln", FP32, _lap_rows(), cols, offset=1e3, seed=2)


@pytest.mark.parametrize("dtype,cols", [(BF16, 1000), (BF16, 11008), (FP16, 5120), (FP32, 2056)])
def test_rms_norm_residual_grads_through_y_and_h(dtype, cols):
    """y, h = rms_norm(x, w, residual=r): h = x + r rounded to dtype and y = rmsnorm(h) * w; gradients flow into x and r
    from both outputs (dx = dr = d(norm)/dh + dh)."""
    torch.manual_seed(3)
    rows = _lap_rows()
    x = torch.randn(rows, cols, device="cuda").to(dtype).requires_grad_(True)
    res = torch.randn(rows, cols, device="cuda").to(dtype).requires_grad_(True)
    w = (torch.rand(cols, device="cuda") + 0.5).to(dtype).requires_grad_(True)
    y, h = launches(lambda: KN.rms_norm(x, w, 1e-6, residual=res))
    y, h = _t(y), _t(h)
    assert torch.equal(h, (x.detach().float() + res.detach().float()).to(dtype))
    gy, gh = torch.randn_like(y), torch.randn_like(h)
    ((y.float() * gy.float()).sum() + (h.float() * gh.float()).sum()).backward()

    h64 = h.detach().double().requires_grad_(True)      # the kernel normalises the stored (rounded) h
    w64 = w.detach().double().requires_grad_(True)
    r = torch.rsqrt(h64.pow(2).mean(-1, keepdim=True) + 1e-6)
    y64 = h64 * r * w64
    ((y64 * gy.double()).sum() + (h64 * gh.double()).sum()).backward()
    rt = RTOL[dtype]
    tag = f"rms+residual {str(dtype)[6:]} {rows}x{cols}"
    check(f"{tag} y", y, y64, rt)
    # dx = round(round(d_norm) + gh): two roundings, bounded against the magnitude of both terms
    gw = gy.double() * w64.detach()
    xh = (h64 * r).detach()
    d_norm = h64.grad - gh.double()
    mag = rt * d_norm.abs() + K_SUM * U32 * r.detach() * (gw.abs() + xh.abs() * (gw * xh).abs().mean(-1, keepdim=True))
    check(f"{tag} dx", x.grad, h64.grad, rt, mag)
    check(f"{tag} dresidual", res.grad, h64.grad, rt, mag)
    check(f"{tag} dw", w.grad, w64.grad, rt, K_SUM * U32 * (gy.double().abs() * xh.abs()).sum(0))


# ------------------------------------------------------------------------------------------------ fused cross-entropy
CE_DTYPES = [BF16, FP16, FP32]
CE_VOCABS = [32000, 50257, 128256, 1003]   # vector path, all scalar tail, Llama-3, tiny (tail)
CE_RTOL32 = 1e-5                           # fp32 gradients: __expf is (2 + 1.16|x|) ulp, |x - lse| <= ~25 here
CE_LSE_ATOL = K_SUM * U32                  # lse = m + log(sum of __expf terms), an absolute error of a few fp32 steps


def _vec(dtype):
    return 16 // torch.tensor([], dtype=dtype).element_size()


def _ce_labels(rows, vocab, ignore):
    lab = torch.randint(0, vocab, (rows,), device="cuda")
    lab[0], lab[1], lab[2], lab[3] = 0, vocab - 1, vocab - 3, ignore   # first column, last column, the row's tail, ignored
    return lab


def _ce_ref_check(tag, lg, lab, ignore, loss, grad, dloss, dtype):
    x = lg.detach().double()
    ref = F.cross_entropy(x, lab, ignore_index=ignore, reduction="none")
    lse = torch.logsumexp(x, -1)
    valid = lab != ignore
    xl = torch.where(valid, x.gather(1, lab.clamp(min=0)[:, None]).squeeze(1), torch.zeros_like(lse))
    # loss = lse - x[label] cancels; lse carries the absolute error of the log of an fp32 sum of __expf terms
    atol = (CE_LSE_ATOL + 2 * U32 * (lse.abs() + xl.abs())) * valid
    check(f"{tag} loss", loss, ref, 2 * U32, atol)
    p = torch.softmax(x, -1)
    onehot = torch.zeros_like(p)
    onehot[valid, lab[valid]] = 1.0
    gref = (p - onehot) * (dloss.double() * valid)[:, None]
    rt = RTOL[dtype] if dtype != FP32 else CE_RTOL32
    check(f"{tag} grad", grad, gref, rt, CE_RTOL32 * (p + onehot) * dloss.double().abs()[:, None])


@pytest.mark.parametrize("vocab", CE_VOCABS)
@pytest.mark.parametrize("dtype", CE_DTYPES)
def test_softmax_ce_elementwise(dtype, vocab):
    """Loss, lse and gradient of KL.softmax_cross_entropy, out of place and in place (the gradient overwrites the logits:
    llama.py, gpt.py and mixtral.py train that way); the in-place gradient equals the out-of-place one bit for bit."""
    torch.manual_seed(4)
    rows, ignore = 67, -100
    base = (torch.randn(rows, vocab, device="cuda") * 3).to(dtype)
    lab = _ce_labels(rows, vocab, ignore)
    dloss = torch.rand(rows, device="cuda") + 0.5
    lg = base.clone().requires_grad_(True)
    loss = launches(lambda: _t(KL.softmax_cross_entropy(lg, lab, ignore)))
    (loss * dloss).sum().backward()
    tag = f"ce {str(dtype)[6:]} V={vocab}"
    _ce_ref_check(tag, lg, lab, ignore, loss, lg.grad, dloss, dtype)
    _, lse = _ext().softmax_ce_fwd(base, lab, ignore)
    x = base.double()
    check(f"{tag} lse", lse, torch.logsumexp(x, -1), 2 * U32, CE_LSE_ATOL)

    leaf = base.clone().requires_grad_(True)
    act = leaf * 1                                     # a non-leaf logits tensor, as a model's head output
    loss_ip = _t(KL.softmax_cross_entropy(act, lab, ignore, inplace_backward=True))
    assert torch.equal(loss_ip, loss)
    (loss_ip * dloss).sum().backward()
    assert torch.equal(leaf.grad, lg.grad)
    assert torch.equal(act.detach(), lg.grad)          # the gradient was written over the logits
    # the binding: the in-place result is the logits tensor itself
    buf = base.clone()
    _, lse = _ext().softmax_ce_fwd(buf, lab, ignore)
    out = _ext().softmax_ce_bwd(buf, lab, lse, dloss, ignore, True)
    assert out.data_ptr() == buf.data_ptr() and torch.equal(buf, lg.grad)


def _mask_runs(x, vocab, n):
    """-inf over aligned n-wide runs at several offsets (rows 4..7) and over the second half of row 8."""
    nvec = vocab // n
    starts = sorted({0, (nvec * 3 // 20) * n, (nvec * 3 // 4) * n, (nvec - 1) * n})
    for i, s in enumerate(starts):
        x[4 + i % 4, s:s + n] = float("-inf")
        x[4 + (i + 1) % 4, s:s + n] = float("-inf")
    x[8, vocab // 2:] = float("-inf")
    return x


@pytest.mark.parametrize("vocab", CE_VOCABS)
@pytest.mark.parametrize("dtype", CE_DTYPES)
def test_softmax_ce_masked_logits(dtype, vocab):
    """Vocabulary ids masked to -inf (padded vocab, constrained targets): aligned 8-wide (16-bit) / 4-wide (fp32) runs and
    a masked half-row keep loss and gradient finite and equal to float64 F.cross_entropy; masked ids get an exact 0."""
    torch.manual_seed(5)
    rows, ignore = 16, -100
    x = _mask_runs((torch.randn(rows, vocab, device="cuda") * 3).to(dtype), vocab, _vec(dtype))
    masked = torch.isinf(x)
    lab = torch.randint(0, vocab // 2, (rows,), device="cuda")
    lab = torch.where(masked.gather(1, lab[:, None]).squeeze(1), lab + 8, lab)   # labels on unmasked ids (runs are <= 8 wide)
    assert not masked.gather(1, lab[:, None]).any()
    lab[3] = ignore
    dloss = torch.rand(rows, device="cuda") + 0.5
    lg = x.clone().requires_grad_(True)
    loss = _t(KL.softmax_cross_entropy(lg, lab, ignore))
    (loss * dloss).sum().backward()
    assert torch.isfinite(loss).all(), loss
    assert torch.isfinite(lg.grad).all()
    assert (lg.grad[masked] == 0).all()
    _ce_ref_check(f"ce masked {str(dtype)[6:]} V={vocab}", lg, lab, ignore, loss, lg.grad, dloss, dtype)


def test_softmax_ce_fully_masked_row_stays_nan():
    """A row that is -inf everywhere has no distribution: lse -inf and loss NaN, as torch gives."""
    x = torch.randn(4, 32000, device="cuda").to(BF16)
    x[2] = float("-inf")
    lab = torch.tensor([1, 2, 3, 4], device="cuda")
    loss, lse = _ext().softmax_ce_fwd(x, lab, -100)
    assert lse[2].item() == float("-inf") and math.isnan(loss[2].item())
    assert torch.isfinite(loss[[0, 1, 3]]).all()
    assert torch.isnan(F.cross_entropy(x.double(), lab, reduction="none")[2])


# ------------------------------------------------------------------------------------------------ vocab-parallel cross-entropy
@pytest.mark.parametrize("widths", [(12005, 19995), (8000, 7997, 8011, 7992)], ids=["2shards", "4shards"])
@pytest.mark.parametrize("dtype", CE_DTYPES)
def test_vocab_parallel_ce_on_one_gpu(dtype, widths):
    """vp_ce_max / vp_ce_sumexp / vp_ce_bwd per vocab shard, with the max and sum all-reduces done by hand as
    _VocabParallelCE.forward does them, against the float64 full-vocabulary cross-entropy.  Shard widths are uneven and
    some are not a multiple of the 16-byte vector (scalar rows)."""
    torch.manual_seed(6)
    rows, ignore, vocab = 24, -100, sum(widths)
    starts = [sum(widths[:i]) for i in range(len(widths))]
    x = (torch.randn(rows, vocab, device="cuda") * 3).to(dtype)
    lab = torch.randint(0, vocab, (rows,), device="cuda")
    for i, s in enumerate(starts):                      # a label in every shard, at its first and last id
        lab[2 * i], lab[2 * i + 1] = s, s + widths[i] - 1
    lab[2 * len(widths)] = ignore
    n = _vec(dtype)
    r = 2 * len(widths) + 1
    x[r, 8 * n:16 * n] = float("-inf")                  # an aligned masked run inside the first shard
    lab[r] = starts[-1] + 5
    x[r + 1, starts[1]:starts[1] + widths[1]] = float("-inf")   # one shard wholly masked for a row
    lab[r + 1] = starts[0]
    dloss = torch.rand(rows, device="cuda") + 0.5
    shards = [x[:, s:s + w].contiguous() for s, w in zip(starts, widths)]
    E = _ext()
    row_max = torch.stack([E.vp_ce_max(sh) for sh in shards]).amax(0)
    parts = [E.vp_ce_sumexp(sh, lab, row_max, s) for sh, s in zip(shards, starts)]
    sumexp = torch.stack([p[0] for p in parts]).sum(0)
    tgt = torch.stack([p[1] for p in parts]).sum(0)
    loss = torch.log(sumexp) + row_max - tgt
    loss = torch.where(lab == ignore, torch.zeros_like(loss), loss)
    grad = torch.cat([E.vp_ce_bwd(sh, lab, row_max, sumexp, dloss, s, ignore, False) for sh, s in zip(shards, starts)], 1)
    assert torch.isfinite(loss).all() and torch.isfinite(grad).all()
    assert (grad[torch.isinf(x)] == 0).all()
    assert torch.equal(row_max, x.float().amax(-1))
    _ce_ref_check(f"vp-ce {str(dtype)[6:]} {len(widths)} shards", x, lab, ignore, loss, grad, dloss, dtype)


# ------------------------------------------------------------------------------------------------ rotary
def _rope64(x, cos, sin, pos, neox):
    """float64 rotary on [B, S, H, D]; tables [P, D/2]; pos [B, S] or None (position = index in the sequence)."""
    b, s, h, d = x.shape
    if pos is None:
        pos = torch.arange(s, device=x.device).expand(b, s)
    c, sn = cos[pos][:, :, None, :], sin[pos][:, :, None, :]
    if neox:
        a, bb = x[..., : d // 2], x[..., d // 2:]
        return torch.cat([a * c - bb * sn, bb * c + a * sn], -1), torch.cat([(a * c).abs() + (bb * sn).abs()] * 2, -1)
    a, bb = x[..., 0::2], x[..., 1::2]
    mag = (a * c).abs() + (bb * sn).abs() + (bb * c).abs() + (a * sn).abs()
    return torch.stack([a * c - bb * sn, bb * c + a * sn], -1).flatten(-2), torch.stack([mag, mag], -1).flatten(-2)


ROPE_CASES = [(dt, d, neox) for dt in (BF16, FP16, FP32) for d in (64, 128) for neox in (True, False)]


@pytest.mark.parametrize("pos_ids", [False, True], ids=["seqpos", "position_ids"])
@pytest.mark.parametrize("dtype,dim,neox", ROPE_CASES)
def test_rope_elementwise(dtype, dim, neox, pos_ids):
    """KR.apply_rope forward and backward (the inverse rotation) against float64 autograd; explicit position_ids are
    non-monotonic and repeat."""
    torch.manual_seed(7)
    b, s, h = 2, 96, 5
    cos, sin = KR.rope_tables(4 * s, dim, device="cuda")
    pos = torch.randint(0, 4 * s, (b, s), device="cuda") if pos_ids else None
    if pos is not None:
        pos[:, 10:20] = pos[:, :10]                      # repeats
    x = torch.randn(b, s, h, dim, device="cuda").to(dtype).requires_grad_(True)
    y = launches(lambda: _t(KR.apply_rope(x, cos, sin, pos, neox)))
    dy = torch.randn_like(y)
    y.backward(dy)
    x64 = x.detach().double().requires_grad_(True)
    y64, mag = _rope64(x64, cos.double(), sin.double(), pos, neox)
    y64.backward(dy.double())
    tag = f"rope {str(dtype)[6:]} d={dim} {'neox' if neox else 'interleaved'}{' pos' if pos_ids else ''}"
    check(f"{tag} y", y, y64, RTOL[dtype], 4 * U32 * mag.detach())
    _, gmag = _rope64(dy.double(), cos.double(), sin.double(), pos, neox)
    check(f"{tag} dx", x.grad, x64.grad, RTOL[dtype], 4 * U32 * gmag)


@pytest.mark.parametrize("dtype,dim,neox", [(BF16, 128, True), (FP16, 64, False), (FP32, 128, False), (BF16, 64, True)])
def test_rope_packed_rotates_q_k_and_keeps_v(dtype, dim, neox):
    """KR.apply_rope_packed / rope_packed_ on a [B, S, nh + 2*nkv, D] QKV tensor with GQA head counts: q and k heads match
    float64, v heads are bit-identical to the input, and the gradient w.r.t. the packed tensor matches float64 autograd."""
    torch.manual_seed(8)
    b, s, nh, nkv = 2, 80, 8, 2
    total, rope_heads = nh + 2 * nkv, nh + nkv
    cos, sin = KR.rope_tables(2 * s, dim, device="cuda")
    pos = torch.randint(0, 2 * s, (b, s), device="cuda")
    leaf = torch.randn(b, s, total, dim, device="cuda").to(dtype).requires_grad_(True)
    qkv = leaf.clone()
    before = qkv.detach().clone()
    out = launches(lambda: _t(KR.apply_rope_packed(qkv, cos, sin, rope_heads, total, dim, pos, neox=neox)))
    g = torch.randn_like(out)
    out.backward(g)
    assert torch.equal(out[:, :, rope_heads:], before[:, :, rope_heads:])
    x64 = before.double().requires_grad_(True)
    rot, mag = _rope64(x64[:, :, :rope_heads], cos.double(), sin.double(), pos, neox)
    y64 = torch.cat([rot, x64[:, :, rope_heads:]], 2)
    y64.backward(g.double())
    tag = f"rope_packed {str(dtype)[6:]} d={dim} {'neox' if neox else 'interleaved'}"
    check(f"{tag} qk", out[:, :, :rope_heads], rot, RTOL[dtype], 4 * U32 * mag.detach())
    _, gmag = _rope64(g.double()[:, :, :rope_heads], cos.double(), sin.double(), pos, neox)
    check(f"{tag} dqk", leaf.grad[:, :, :rope_heads], x64.grad[:, :, :rope_heads], RTOL[dtype], 4 * U32 * gmag)
    assert torch.equal(leaf.grad[:, :, rope_heads:], g[:, :, rope_heads:])


# ------------------------------------------------------------------------------------------------ SwiGLU
SWIGLU_ATOL = 1e-30   # silu(x) for x < -87: e^-x overflows fp32 and the kernel's sigmoid is 0; the true value is < 1e-36


@pytest.mark.parametrize("packed", [False, True], ids=["split", "packed"])
@pytest.mark.parametrize("dtype", [BF16, FP16, FP32])
def test_swiglu_elementwise(dtype, packed):
    """KA.swiglu split and packed, forward and backward, with a row count whose vector count is not a multiple of
    grid * 256 * U (the unrolled loop's tail) and gate values up to |x| = 100, where __expf(-x) saturates."""
    torch.manual_seed(9)
    cols = 1024
    n = _vec(dtype)
    vec_rows = cols // n
    grid = _sms() * 16
    rows = (grid * 256 * 4) // vec_rows + 3                 # one full unrolled lap of the forward grid and a ragged tail
    gate = torch.randn(rows, cols, device="cuda") * 4
    gate[:, :64] = torch.linspace(-100, 100, 64, device="cuda")
    up = torch.randn(rows, cols, device="cuda")
    gate, up = gate.to(dtype), up.to(dtype)
    if packed:
        xin = torch.cat([gate, up], -1).requires_grad_(True)
        y = launches(lambda: _t(KA.swiglu(xin)))
    else:
        g_, u_ = gate.clone().requires_grad_(True), up.clone().requires_grad_(True)
        y = launches(lambda: _t(KA.swiglu(g_, u_)))
    dy = torch.randn_like(y)
    y.backward(dy)
    g64, u64 = gate.double().requires_grad_(True), up.double().requires_grad_(True)
    y64 = F.silu(g64) * u64
    y64.backward(dy.double())
    sg = torch.sigmoid(g64.detach())
    tag = f"swiglu {str(dtype)[6:]} {'packed' if packed else 'split'}"
    rt = RTOL[dtype] if dtype != FP32 else 2e-5             # __expf(-x) is (2 + 1.16|x|) ulp up to |x| = 100
    assert torch.isfinite(y).all()
    check(f"{tag} y", y, y64, rt, SWIGLU_ATOL)
    dg, du = (xin.grad[:, :cols], xin.grad[:, cols:]) if packed else (g_.grad, u_.grad)
    assert torch.isfinite(dg).all() and torch.isfinite(du).all()
    # d gate = dy * y * sg * (1 + x (1 - sg)) cancels at x ~ -1.28
    mag = (dy.double() * u64.detach() * sg).abs() * (1 + (g64.detach() * (1 - sg)).abs())
    check(f"{tag} dgate", dg, g64.grad, rt, SWIGLU_ATOL + 64 * U32 * mag)
    check(f"{tag} dup", du, u64.grad, rt, SWIGLU_ATOL)


# ------------------------------------------------------------------------------------------------ optimizers
def _f32(v):
    return float(torch.tensor(v, dtype=FP32))


# hyper-parameters as the kernels receive them (fp32), so the float64 references use the same values
B1, B2, EPS, WD, LR = (_f32(v) for v in (0.9, 0.95, 1e-8, 0.1, 1e-2))


def _slab(n, dtype, offset, fill):
    """A contiguous n-element tensor; offset=1 makes it a view one element into its buffer (not 16-byte aligned)."""
    buf = torch.empty(n + offset, device="cuda", dtype=dtype)
    t = buf[offset:]
    t.copy_(fill)
    return t


def _adamw_ref(p, g, m, v, step, gscale, lr=LR):
    """float64 AdamW (decoupled weight decay, bias-corrected) and the magnitude of the terms each output sums; the
    parameter's magnitude includes the fp32 error of m, which cancels when B1 m ~ -(1 - B1) g."""
    bc1, bc2 = _f32(1 - B1 ** step), _f32(1 - B2 ** step)
    gg = g * gscale
    m1 = B1 * m + (1 - B1) * gg
    v1 = B2 * v + (1 - B2) * gg * gg
    denom = v1.sqrt() / math.sqrt(bc2) + EPS
    upd = lr / bc1 * m1 / denom
    p1 = p * (1 - lr * WD) - upd
    mmag = (B1 * m).abs() + ((1 - B1) * gg).abs()
    return p1, m1, v1, (p * (1 - lr * WD)).abs() + upd.abs() + lr / bc1 * mmag / denom, mmag


ADAMW_TYPES = [(FP32, FP32, False), (BF16, BF16, True), (BF16, FP32, True), (FP16, FP16, True), (FP16, FP32, True),
               (BF16, BF16, False)]


@pytest.mark.parametrize("aligned", [True, False], ids=["vector", "scalar"])
@pytest.mark.parametrize("state", [FP32, BF16])
@pytest.mark.parametrize("p_dt,g_dt,master", ADAMW_TYPES)
def test_adamw_steps_against_float64(p_dt, g_dt, master, state, aligned):
    """adamw_step for three steps, each against the float64 update of the kernel's own inputs: the 16-byte vector kernel
    with a scalar tail (n = 8k + 5), and the scalar kernel on slabs one element off alignment."""
    torch.manual_seed(10)
    n, off = 8 * 4099 + 5, 0 if aligned else 1
    p0 = torch.randn(n, device="cuda")
    p = _slab(n, p_dt, off, p0.to(p_dt))
    mst = _slab(n, FP32, off, p.float()) if master else None
    m = _slab(n, state, off, torch.zeros(n, device="cuda"))
    v = _slab(n, state, off, torch.zeros(n, device="cuda"))
    E = _ext()
    for step in (1, 2, 3):
        g = _slab(n, g_dt, off, (torch.randn(n, device="cuda") * 0.1).to(g_dt))
        pin = (mst if master else p).double()
        min_, vin = m.double(), v.double()
        E.adamw_step(p, g, mst, m, v, LR, B1, B2, EPS, WD, step, None, 0.0, None, None)
        p1, m1, v1, pmag, mmag = _adamw_ref(pin, g.double(), min_, vin, step, 1.0)
        tag = f"adamw p={str(p_dt)[6:]} g={str(g_dt)[6:]} state={str(state)[6:]} {'vec' if aligned else 'scalar'} step {step}"
        check(f"{tag} m", m, m1, RTOL[state], 4 * U32 * mmag)
        check(f"{tag} v", v, v1, RTOL[state])
        if master:
            check(f"{tag} master", mst, p1, RTOL[FP32], 8 * U32 * pmag)
        check(f"{tag} p", p, p1, RTOL[p_dt], 8 * U32 * pmag)


@pytest.mark.parametrize("case", ["found_inf", "inv_scale", "clip_active", "clip_inactive"])
def test_adamw_found_inf_unscale_and_clip(case):
    """The device-side arguments of adamw_step: found_inf set leaves every tensor bit-identical; inv_scale unscales the
    gradient; grad_sq_norm with max_norm below the norm scales it by max_norm / (norm + 1e-6), above leaves it."""
    torch.manual_seed(11)
    n = 8 * 5000 + 3
    p = (torch.randn(n, device="cuda")).to(BF16)
    mst, m, v = p.float(), torch.rand(n, device="cuda") * 0.01, torch.rand(n, device="cuda") * 1e-4
    loss_scale = 1024.0 if case == "inv_scale" else 1.0
    g_true = torch.randn(n, device="cuda") * 0.1
    g = (g_true * loss_scale).to(BF16)
    gsq = (g.double() ** 2).sum()
    norm = math.sqrt(gsq.item()) / loss_scale
    fi = torch.tensor([1.0 if case == "found_inf" else 0.0], device="cuda")
    inv = torch.tensor([1.0 / loss_scale], device="cuda")
    sq = torch.tensor([gsq.item()], device="cuda", dtype=FP32)
    max_norm = {"clip_active": norm / 3, "clip_inactive": norm * 3}.get(case, 0.0)
    before = [t.clone() for t in (p, mst, m, v)]
    _ext().adamw_step(p, g, mst, m, v, LR, B1, B2, EPS, WD, 4, sq if max_norm else None, max_norm, fi, inv)
    if case == "found_inf":
        for a, b in zip((p, mst, m, v), before):
            assert torch.equal(a, b)
        return
    gscale = 1.0 / loss_scale
    if case == "clip_active":
        gscale *= max_norm / (math.sqrt(float(sq.item())) / loss_scale + 1e-6)
    p1, m1, v1, pmag, mmag = _adamw_ref(before[1].double(), g.double(), before[2].double(), before[3].double(), 4, gscale)
    check(f"adamw {case} m", m, m1, RTOL[FP32], 4 * U32 * mmag)
    check(f"adamw {case} v", v, v1, RTOL[FP32])
    check(f"adamw {case} master", mst, p1, RTOL[FP32], 8 * U32 * pmag)
    check(f"adamw {case} p", p, p1, RTOL[BF16], 8 * U32 * pmag)


@pytest.mark.parametrize("aligned", [True, False], ids=["vector", "scalar"])
def test_adamw_step_dyn_is_bit_equal_to_adamw_step(aligned):
    """The graph-capturable adamw_step_dyn, with dyn = {lr, 1 - b1^t, 1 - b2^t} on the device, computes exactly what
    adamw_step computes from the same float hyper-parameters."""
    torch.manual_seed(12)
    n, off = 8 * 3001 + 6, 0 if aligned else 1
    p = _slab(n, BF16, off, torch.randn(n, device="cuda").to(BF16))
    ms = _slab(n, FP32, off, p.float())
    m = _slab(n, FP32, off, torch.zeros(n, device="cuda"))
    v = _slab(n, FP32, off, torch.zeros(n, device="cuda"))
    a = [_slab(n, t.dtype, off, t) for t in (p, ms, m, v)]
    E = _ext()
    for step in (1, 2, 3, 4):
        g = (torch.randn(n, device="cuda") * 0.1).to(BF16)
        E.adamw_step(p, g, ms, m, v, LR, B1, B2, EPS, WD, step, None, 0.0, None, None)
        dyn = torch.tensor([LR, 1 - B1 ** step, 1 - B2 ** step], device="cuda", dtype=FP32)
        E.adamw_step_dyn(a[0], g, a[1], a[2], a[3], 1.0, B1, B2, EPS, WD, None, 0.0, None, None, dyn)
        for x, y in zip((p, ms, m, v), a):
            assert torch.equal(x, y), f"step {step}"


@pytest.mark.parametrize("mode", ["plain", "momentum", "nesterov", "master"])
@pytest.mark.parametrize("dtype", [FP32, BF16, FP16])
def test_sgd_step_against_float64(dtype, mode):
    """sgd_step: plain, momentum, Nesterov momentum, and Nesterov with an fp32 master copy, three steps each."""
    torch.manual_seed(13)
    n = 100003
    momentum = 0.0 if mode == "plain" else 0.9
    nesterov = mode in ("nesterov", "master")
    p = torch.randn(n, device="cuda").to(dtype)
    mst = p.float().clone() if mode == "master" else None
    mom = torch.zeros(n, device="cuda") if momentum else None
    lr, wd, momentum = _f32(0.05), _f32(0.01), _f32(momentum)
    for step in range(3):
        g = (torch.randn(n, device="cuda")).to(dtype)
        pin = (mst if mst is not None else p).double()
        min_ = mom.double() if mom is not None else None
        _ext().sgd_step(p, g, mst, mom, lr, momentum, wd, nesterov)
        gf = g.double() + wd * pin
        gmag = g.double().abs() + (wd * pin).abs()
        if mom is not None:
            mv = momentum * min_ + gf
            mvmag = (momentum * min_).abs() + gmag
            check(f"sgd {str(dtype)[6:]} {mode} step {step} mom", mom, mv, RTOL[FP32], 4 * U32 * mvmag)
            gf, gmag = (gf + momentum * mv, gmag + momentum * mvmag) if nesterov else (mv, mvmag)
        p1 = pin - lr * gf
        pmag = pin.abs() + lr * gmag
        if mst is not None:
            check(f"sgd {str(dtype)[6:]} {mode} step {step} master", mst, p1, RTOL[FP32], 4 * U32 * pmag)
        check(f"sgd {str(dtype)[6:]} {mode} step {step} p", p, p1, RTOL[dtype], 4 * U32 * pmag)


def _lamb_ref(p, g, m, v, step, lr, wd):
    bc1, bc2 = _f32(1 - B1 ** step), _f32(1 - B2 ** step)
    m1 = B1 * m + (1 - B1) * g
    v1 = B2 * v + (1 - B2) * g * g
    u = (m1 / bc1) / ((v1 / bc2).sqrt() + EPS) + wd * p
    pn, un = p.norm(), u.norm()
    trust = (pn / un).item() if pn > 0 and un > 0 else 1.0
    return p - lr * trust * u, m1, v1, trust, p.abs() + lr * trust * u.abs()


@pytest.mark.parametrize("param", ["random", "zero"])
@pytest.mark.parametrize("dtype,master", [(FP32, False), (BF16, True), (FP16, True)])
def test_lamb_step_trust_ratio(dtype, master, param):
    """lamb_step: the layer-wise trust ratio ||p|| / ||u|| against float64; a zero parameter has trust ratio 1."""
    torch.manual_seed(14)
    n = 50001
    p = (torch.randn(n, device="cuda") if param == "random" else torch.zeros(n, device="cuda")).to(dtype)
    mst = p.float() if master else None
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    lr, wd = _f32(0.01), _f32(0.01)
    for step in (1, 2, 3):
        g = (torch.randn(n, device="cuda") * 0.1).to(dtype)
        pin = (mst if master else p).double()
        min_, vin = m.double(), v.double()
        _ext().lamb_step(p, g, mst, m, v, lr, B1, B2, EPS, wd, step)
        p1, m1, v1, trust, pmag = _lamb_ref(pin, g.double(), min_, vin, step, lr, wd)
        if param == "zero" and step == 1:
            assert trust == 1.0
        tag = f"lamb {str(dtype)[6:]} {param} step {step}"
        check(f"{tag} m", m, m1, RTOL[FP32], 4 * U32 * ((B1 * min_).abs() + ((1 - B1) * g.double()).abs()))
        check(f"{tag} v", v, v1, RTOL[FP32])
        # the trust ratio comes from two fp32 sums over the whole slab
        tol = RTOL[FP32] + K_SUM * U32
        if master:
            check(f"{tag} master", mst, p1, tol, tol * pmag)
        check(f"{tag} p", p, p1, max(RTOL[dtype], tol), tol * pmag)


@pytest.mark.parametrize("n,offset", [((1 << 20) + 3, 0), (1003, 0), ((1 << 18) + 7, 1)], ids=["tail", "small", "unaligned"])
@pytest.mark.parametrize("dtype", [FP16, BF16, FP32])
def test_grad_sq_norm(dtype, n, offset):
    """grad_sq_norm: sum of squares against float64 (vector body + scalar tail, and the scalar loop of an unaligned
    view); found_inf stays 0 for finite gradients and is set by an inf and by a NaN."""
    torch.manual_seed(15)
    g = _slab(n, dtype, offset, torch.randn(n, device="cuda").to(dtype))
    out, fi = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    _ext().grad_sq_norm(g, out, fi)
    # a sum of positive terms (per-thread loop, block tree, one atomic per CTA): rounding errors do not cancel the value
    check(f"grad_sq_norm {str(dtype)[6:]} n={n} off={offset}", out, (g.double() ** 2).sum().reshape(1), K_SUM * U32)
    assert fi.item() == 0
    for bad in (float("inf"), float("nan")):
        h = g.clone() if offset == 0 else _slab(n, dtype, offset, g)
        h[n - 2] = bad
        out.zero_()
        fi.zero_()
        _ext().grad_sq_norm(h, out, fi)
        assert fi.item() == 1, bad


@pytest.mark.parametrize("dtype", [FP16, BF16, FP32])
def test_scale_inplace_with_device_scale(dtype):
    """scale_inplace(g, scale_dev, scale_host): g *= scale_dev * scale_host, the device scale read inside the kernel."""
    torch.manual_seed(16)
    n = 70001
    g = torch.randn(n, device="cuda").to(dtype)
    scale = torch.tensor([0.37 / 1024], device="cuda")
    ref = g.double() * scale.double() * 0.5
    _ext().scale_inplace(g, scale, 0.5)
    check(f"scale_inplace {str(dtype)[6:]}", g, ref, RTOL[dtype] if dtype != FP32 else 2 * U32)   # fp32: one rounding
