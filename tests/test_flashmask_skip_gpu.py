"""The tile-skipping column-mask kernels (csrc/attention_flashmask_sm100.cu) on the GPU:

1. Bitwise: causal documents on 128-row boundaries, packed into rows, give exactly the bits of each document run alone through the dense
   causal kernels (O, lse, and dQ / dK / dV of the deterministic backward): both walk the same tiles in the same order.
2. float64, within the rounding bound of tests/test_attention_d64_gpu.py (_ref64 / _check_f64), for unaligned documents, random 4-bound
   masks, per-head masks, non-causal calls, sq != sk, rows that see no key and keys no query sees; single pass and deterministic.  The
   kernels that test every element (mask_skip=False, B200_ATTN_MASK_SKIP=0) run on the same inputs and must meet the same bound.
3. Dropout under a document mask: the mask read back exactly, and replayed through fixed_seed_offset.
4. A masked forward + backward captured in a CUDA graph replays the eager results: nothing is read on the host.
5. LlamaForCausalLM on packed documents at head_dim 128 in bf16, on the fused packed path, against each document run alone.
"""
import pytest
import torch

import paddle_b200 as paddle
from paddle_b200.kernels import attention as KAT
from test_attention_d64_gpu import SC, U, _check_f64, _ref64

pytestmark = pytest.mark.gpu

P = 0.3


def _ext():
    from paddle_b200._build import ext

    return ext()


def _det(fn):
    paddle.set_flags({"FLAGS_cudnn_deterministic": True})
    try:
        return fn()
    finally:
        paddle.set_flags({"FLAGS_cudnn_deterministic": False})


def _inputs(b, sq, sk, h, hk, dtype, d, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mk = lambda *s: (torch.randn(*s, device="cuda", generator=g) * 1.5).to(dtype)  # noqa: E731
    return mk(b, sq, h, d), mk(b, sk, hk, d), mk(b, sk, hk, d), mk(b, sq, h, d)


def _docs(rows):
    """Causal document masks of rows of document lengths: int32 [B, 1, S, 4]."""
    ends = [torch.cat([torch.full((n,), e, dtype=torch.int32) for n, e in zip(r, torch.tensor(r).cumsum(0).tolist())]) for r in rows]
    se = torch.stack(ends).reshape(len(rows), 1, -1, 1).cuda()
    return KAT.colmask_from_startend(se, True, se.shape[2])


def _run(q, k, v, g, causal, cm, det, skip=True):
    E = _ext()
    out, lse = E.attention_fwd(q, k, v, SC, causal, False, cm, 0.0, None, skip)
    fn = lambda: E.attention_bwd(q, k, v, out, lse, g, SC, causal, cm, 0.0, None, skip)  # noqa: E731
    dq, dk, dv = _det(fn) if det else fn()
    return out, lse, dq, dk, dv


# ---------------------------------------------------------------------------------------------------- 1. bitwise against documents alone
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d", [64, 128])
def test_aligned_documents_equal_separate_calls(dtype, d):
    rows = [[384, 128, 512], [256, 768]]
    s = 1024
    q, k, v, g = _inputs(2, s, s, 8, 2, dtype, d, seed=d)
    cm = _docs(rows)
    out, lse, dq, dk, dv = _run(q, k, v, g, True, cm, det=True)
    for r, row in enumerate(rows):
        a = 0
        for n in row:
            sl = lambda t: t[r:r + 1, a:a + n].contiguous()  # noqa: E731
            o1, l1, dq1, dk1, dv1 = _run(sl(q), sl(k), sl(v), sl(g), True, None, det=True)
            assert torch.equal(out[r:r + 1, a:a + n], o1), ("out", r, a)
            assert torch.equal(lse[r:r + 1, :, a:a + n], l1), ("lse", r, a)
            assert torch.equal(dq[r:r + 1, a:a + n], dq1), ("dq", r, a)
            assert torch.equal(dk[r:r + 1, a:a + n], dk1), ("dk", r, a)
            assert torch.equal(dv[r:r + 1, a:a + n], dv1), ("dv", r, a)
            a += n


# ---------------------------------------------------------------------------------------------------- 2. float64, and the old kernels
def _mask(kind, b, h, sq, sk, g):
    keys = torch.arange(sk, device="cuda")
    if kind == "docs":            # unaligned documents
        return _docs([[100, 300, 57, sk - 457], [sk]] if b == 2 else [[sk]])
    if kind == "bounds":          # both intervals, varying per key
        lts = (keys * 7 % sq).int()
        lte = (lts + 40 + keys % 90).clamp(max=sq).int()
        uts = (keys % 13).int()
        ute = (uts + (keys * 3 % 150)).clamp(max=sq).int()
        return torch.stack([lts, lte, uts, ute], -1).reshape(1, 1, sk, 4).expand(b, 1, sk, 4).contiguous()
    if kind == "heads":           # a different window per head
        ms = [KAT.colmask_from_window(sq, sk, 30 + 50 * i, 20 * i, False, "cuda") for i in range(h)]
        return torch.cat(ms, 1).expand(b, h, sk, 4).contiguous()
    if kind == "empty":           # rows 130..259 see no key (a whole 128-row tile); keys 256..399 (a whole 128-key tile) no query
        cm = torch.zeros(b, 1, sk, 4, dtype=torch.int32, device="cuda")
        cm[..., 0], cm[..., 1] = 130, 260
        cm[:, :, 256:400, 0], cm[:, :, 256:400, 1] = 0, 2 ** 31 - 1
        return cm
    raise ValueError(kind)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("kind,causal,sq,sk", [("docs", True, 700, 700), ("bounds", False, 555, 690), ("bounds", True, 640, 640),
                                               ("heads", False, 500, 433), ("empty", False, 600, 600), ("empty", True, 600, 600)])
def test_against_float64_and_masked_kernels(dtype, d, kind, causal, sq, sk):
    b, h, hk = 2, 4, 2
    q, k, v, g = _inputs(b, sq, sk, h, hk, dtype, d, seed=sq + d)
    cm = _mask(kind, b, h, sq, sk, g)
    vis = KAT.colmask_to_dense(cm, sq)
    ref, bnd = _ref64(q, k, v, g, causal, vis)
    for det in (False, True):
        new = _run(q, k, v, g, causal, cm, det)
        old = _run(q, k, v, g, causal, cm, det, skip=False)
        print(kind, "det" if det else "one-pass", "float64 worst: new", _check_f64(new, q, k, v, g, causal, vis), "old",
              _check_f64(old, q, k, v, g, causal, vis))
        for name, a, c, bd in zip(("out", "dq", "dk", "dv"), (new[0], new[2], new[3], new[4]), (old[0], old[2], old[3], old[4]),
                                  (bnd[0], bnd[2], bnd[3], bnd[4])):
            assert ((a.double() - c.double()).abs() <= 4 * bd).all(), name
    if kind == "empty":
        out, lse, dq, dk, dv = new
        assert torch.all(out[:, 130:260] == 0) and torch.all(lse[:, :, 130:260] == float("-inf")) and torch.all(dq[:, 130:260] == 0)
        assert torch.all(dk[:, 256:400] == 0) and torch.all(dv[:, 256:400] == 0)
        for t in (out, dq, dk, dv):
            assert torch.isfinite(t).all()


def test_single_pass_matches_deterministic():
    q, k, v, g = _inputs(2, 1000, 1000, 8, 2, torch.bfloat16, 128, seed=9)
    cm = _mask("docs", 2, 8, 1000, 1000, None)
    one, det = _run(q, k, v, g, True, cm, False), _run(q, k, v, g, True, cm, True)
    for i in (0, 1, 3, 4):                 # O, lse, and dK / dV (accumulated in registers in a fixed order) are the same bits
        assert torch.equal(one[i], det[i]), i
    ref, bnd = _ref64(q, k, v, g, True, KAT.colmask_to_dense(cm, 1000))
    assert ((one[2].double() - det[2].double()).abs() <= 4 * bnd[2]).all()


# ---------------------------------------------------------------------------------------------------- 3. dropout under documents
@pytest.mark.parametrize("d", [64, 128])
def test_dropout_mask_readout_with_documents(d):
    b, h, hk, s, dtype = 2, 4, 2, 200, torch.bfloat16
    q = torch.zeros(b, s, h, d, dtype=dtype, device="cuda")
    k = torch.zeros(b, s, hk, d, dtype=dtype, device="cuda")
    v = torch.zeros(b, s, hk, d, dtype=dtype, device="cuda")
    v[:, torch.arange(min(s, d)), :, torch.arange(min(s, d))] = 1       # V[j] = e_j for the keys j < d
    cm = _docs([[37, 90, 73], [128, 72]])
    E = _ext()
    out, lse, so = E.attention_fwd(q, k, v, 0.125, True, False, cm, P, None)
    vis = (torch.ones(s, s, dtype=torch.bool, device="cuda").tril()[None, None] & KAT.colmask_to_dense(cm, s)).expand(b, h, s, s)
    sd, od = (int(x) for x in so.cpu())
    z = KAT.dropout_keep_mask(sd, od, b, h, s, s, P, device="cuda")
    n = min(s, d)
    o = out[..., :n].permute(0, 2, 1, 3)
    assert torch.equal(o != 0, (z & vis)[..., :n])
    cnt = vis.sum(-1, keepdim=True).clamp(min=1).double()
    refv = (z & vis)[..., :n].double() / ((1 - P) * cnt)
    assert ((o.double() - refv).abs() <= U[dtype] * refv + 1e-30).all()
    again = E.attention_fwd(q, k, v, 0.125, True, False, cm, P, so.cpu())
    assert torch.equal(again[0], out) and torch.equal(again[2].cpu(), so.cpu())


# ---------------------------------------------------------------------------------------------------- 4. CUDA graph capture
def test_capture_replays_eager_results():
    q, k, v, g = _inputs(2, 700, 700, 8, 2, torch.bfloat16, 128, seed=4)
    cm = _mask("docs", 2, 8, 700, 700, None)
    eager = _run(q, k, v, g, True, cm, True)
    paddle.set_flags({"FLAGS_cudnn_deterministic": True})
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            _run(q, k, v, g, True, cm, False)                             # warm-up on the capture stream
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            res = _run(q, k, v, g, True, cm, False)
        for x in (q, k, v, g):
            x.mul_(1.0)
        graph.replay()
        torch.cuda.synchronize()
    finally:
        paddle.set_flags({"FLAGS_cudnn_deterministic": False})
    for a, e in zip(res, eager):
        assert torch.equal(a, e)


# ---------------------------------------------------------------------------------------------------- 5. Llama on packed documents
def test_llama_documents_match_separate_runs(monkeypatch):
    from paddle_b200.models import LlamaForCausalLM, llama_tiny

    def no_ref(*a, **kw):
        raise AssertionError("attention fell back to the reference path")

    paddle.set_device("gpu:0")
    paddle.set_default_dtype("bfloat16")
    try:
        paddle.seed(0)
        cfg = llama_tiny(hidden_size=512, intermediate_size=1024, num_attention_heads=4, num_key_value_heads=2, num_hidden_layers=2,
                         vocab_size=1024, max_position_embeddings=1024)
        model = LlamaForCausalLM(cfg)
        model.train()
        rows = [[256, 128, 384, 256], [1024]]
        s = 1024
        gen = torch.Generator(device="cuda").manual_seed(3)
        ids = torch.randint(0, cfg.vocab_size, (2, s + 1), device="cuda", generator=gen)
        x, y = ids[:, :-1], ids[:, 1:].clone()
        for r, row in enumerate(rows):
            for e in torch.tensor(row).cumsum(0).tolist()[:-1]:
                y[r, e - 1] = -100
        ends = torch.stack([torch.cat([torch.full((n,), e) for n, e in zip(row, torch.tensor(row).cumsum(0).tolist())]) for row in rows])
        pos = torch.stack([torch.cat([torch.arange(n) for n in row]) for row in rows]).cuda()
        se = ends.reshape(2, 1, s, 1).int().cuda()
        Pt = lambda t: t.as_subclass(paddle.Tensor)  # noqa: E731
        seen = []
        orig = KAT._FlashAttnPacked.forward

        def fwd(ctx, *a):
            seen.append(a[-1] is not None)
            return orig(ctx, *a)

        monkeypatch.setattr(KAT._FlashAttnPacked, "forward", staticmethod(fwd))
        monkeypatch.setattr(KAT, "attention_ref", no_ref)
        loss = model(Pt(x), Pt(y), Pt(pos), Pt(se))
        loss.backward()
        assert seen and all(seen), "the documents did not take the fused packed path"
        packed = {n: p.grad.as_subclass(torch.Tensor).float().clone() for n, p in model.named_parameters()}
        model.clear_gradients()
        total, n_tok = 0.0, 0
        for r, row in enumerate(rows):
            a = 0
            for n in row:
                xi, yi = x[r:r + 1, a:a + n], y[r:r + 1, a:a + n]
                valid = int((yi != -100).sum())
                li = model(Pt(xi), Pt(yi))
                (li.float() * valid).backward()
                total += float(li) * valid
                n_tok += valid
                a += n
        print(f"loss packed {float(loss):.6f} separate {total / n_tok:.6f}")
        assert abs(float(loss) - total / n_tok) <= 2e-2 * abs(total / n_tok)
        worst = 0.0
        for name, gp in packed.items():
            gs = dict(model.named_parameters())[name].grad.as_subclass(torch.Tensor).float() / n_tok
            rel = ((gp - gs).norm() / gs.norm().clamp(min=1e-12)).item()
            worst = max(worst, rel)
            assert rel < 5e-2, (name, rel)
        print(f"worst relative gradient difference {worst:.4f}")
    finally:
        paddle.set_default_dtype("float32")


# ---------------------------------------------------------------------------------------------------- routing
@pytest.mark.parametrize("skip", [True, False])
def test_switch_routes_masked_calls(skip, monkeypatch):
    """Column-masked calls run the skipping kernels, or with the switch off the kernels that test every element."""
    monkeypatch.setattr(KAT, "_mask_skip", [skip])
    q, k, v, g = (t.requires_grad_(True) if i < 3 else t for i, t in enumerate(_inputs(2, 700, 700, 4, 2, torch.bfloat16, 128, seed=1)))
    cm = _mask("docs", 2, 4, 700, 700, None)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        out = KAT.attention_colmask(q, k, v, cm, causal=True)
        torch.autograd.backward(out.as_subclass(torch.Tensor), g)
        torch.cuda.synchronize()
    names = " ".join(e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    for kern in ("fwd_skip_kernel", "dkv_skip_kernel", "mask_tiles_kernel"):
        assert (kern in names) == skip, kern
    assert ("fwd_kernel" in names) != skip
