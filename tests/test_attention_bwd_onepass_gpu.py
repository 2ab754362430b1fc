"""The single-pass attention backward (dQ bulk-reduced from the dK/dV kernel) against autograd of an fp32 reference and against the
deterministic two-kernel path (FLAGS_cudnn_deterministic), on the shapes and layouts the kernels serve: causal or not, GQA, sequence
lengths that are not tile multiples, a column mask, the packed sequence-major layout, fp16 and the Llama-2-7B training shape."""
import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import kernels
from paddle_b200.kernels import attention as KAT

pytestmark = pytest.mark.gpu


def _ext():
    from paddle_b200._build import ext

    return ext()


def rel_err(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp(min=1e-12)).item()


def _ref(q, k, v, causal, vis=None):
    """fp32 attention on [B,S,H,D]; vis: boolean visibility [B, 1|H, Sq, Sk]."""
    h, hk = q.shape[2], k.shape[2]
    if hk != h:
        k, v = k.repeat_interleave(h // hk, 2), v.repeat_interleave(h // hk, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * q.shape[-1] ** -0.5
    if causal:
        s = s.masked_fill(~torch.ones(q.shape[1], k.shape[1], dtype=torch.bool, device=q.device).tril(), float("-inf"))
    if vis is not None:
        s = s.masked_fill(~vis, float("-inf"))
    return torch.einsum("bhqk,bkhd->bqhd", s.softmax(-1), v)


def _deterministic(fn):
    paddle.set_flags({"FLAGS_cudnn_deterministic": True})
    try:
        return fn()
    finally:
        paddle.set_flags({"FLAGS_cudnn_deterministic": False})


def _check(b, s, h, hk, causal, dtype=torch.bfloat16, colmask=None, vis=None):
    E = _ext()
    torch.manual_seed(7)
    q = (torch.randn(b, s, h, 128, device="cuda") * 0.8).to(dtype)
    k = (torch.randn(b, s, hk, 128, device="cuda") * 0.8).to(dtype)
    v = (torch.randn(b, s, hk, 128, device="cuda") * 0.8).to(dtype)
    g = torch.randn(b, s, h, 128, device="cuda").to(dtype)
    sc = 128 ** -0.5
    out, lse = E.attention_fwd(q, k, v, sc, causal, False, colmask)
    kernels.reset_launch_count()
    one = E.attention_bwd(q, k, v, out, lse, g, sc, causal, colmask)
    assert kernels.launch_count() == 2                 # stats / dQ zeroing + the single pass
    kernels.reset_launch_count()
    det = _deterministic(lambda: E.attention_bwd(q, k, v, out, lse, g, sc, causal, colmask))
    assert kernels.launch_count() == 3                 # stats + dK/dV + dQ
    q32, k32, v32 = (t.float().requires_grad_(True) for t in (q, k, v))
    _ref(q32, k32, v32, causal, vis).backward(g.float())
    for name, a, c, r in zip(("dq", "dk", "dv"), one, det, (q32.grad, k32.grad, v32.grad)):
        assert a.dtype == dtype and a.shape == r.shape, name
        assert rel_err(a, r) < 2e-2, (name, rel_err(a, r))
        assert rel_err(a, c) < 2e-2, (name, "vs deterministic", rel_err(a, c))


@pytest.mark.parametrize("causal", [True, False])
@pytest.mark.parametrize("s", [300, 1000])
@pytest.mark.parametrize("h,hk", [(4, 2), (8, 1)])
def test_onepass_matches_reference_and_deterministic(s, h, hk, causal):
    _check(1, s, h, hk, causal)


def test_onepass_fp16():
    _check(2, 384, 4, 4, True, dtype=torch.float16)


def test_onepass_column_mask():
    b, s, h = 2, 448, 4
    keys = torch.arange(s, device="cuda")
    lts = torch.where(keys < 200, torch.full_like(keys, 200), torch.full_like(keys, s))       # two causal documents per row
    se = lts.reshape(1, 1, s, 1).expand(b, 1, s, 1).int().contiguous()
    cm = KAT.colmask_from_startend(se, True, s).to(torch.int32).contiguous()
    _check(b, s, h, 2, True, colmask=cm, vis=KAT.colmask_to_dense(cm, s))


def test_onepass_packed_seq_major():
    s, b, nh, nkv = 320, 2, 4, 2
    torch.manual_seed(5)
    base = (torch.randn(s, b, nh + 2 * nkv, 128, device="cuda") * 0.7).to(torch.bfloat16)
    g = torch.randn(s, b, nh, 128, device="cuda").to(torch.bfloat16)

    def grad():
        x = base.clone().requires_grad_(True)
        KAT.attention_packed(x, nh, nkv, True, None, seq_major=True).backward(g)
        return x.grad

    one, det = grad(), _deterministic(grad)
    x32 = base.float().transpose(0, 1).requires_grad_(True)
    _ref(x32[:, :, :nh], x32[:, :, nh:nh + nkv], x32[:, :, nh + nkv:], True).backward(g.float().transpose(0, 1))
    ref = x32.grad.transpose(0, 1)
    assert rel_err(one, ref) < 2e-2, rel_err(one, ref)
    assert rel_err(one, det) < 2e-2, rel_err(one, det)


def test_onepass_llama_training_shape():
    _check(1, 4096, 32, 32, True)
