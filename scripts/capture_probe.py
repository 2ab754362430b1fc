"""Which hand-written kernels survive CUDA-graph stream capture? Each op: warm-up eagerly, record into a graph, replay, compare."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import paddle_b200 as paddle  # noqa: E402
from paddle_b200 import _build  # noqa: E402

C = _build.load(required=True)
paddle.set_device("gpu:0")
dev = "cuda"
bf = torch.bfloat16
a = torch.randn(512, 1024, device=dev, dtype=bf)
b = torch.randn(1024, 768, device=dev, dtype=bf)
w = torch.ones(1024, device=dev, dtype=bf)


def probe(name, fn, mode="global"):
    try:
        ref = fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode=mode):
            out = fn()
        g.replay()
        torch.cuda.synchronize()
        o, r = (out[0] if isinstance(out, (list, tuple)) else out), (ref[0] if isinstance(ref, (list, tuple)) else ref)
        print(f"{name:32s} [{mode}] OK  maxdiff={float((o.float() - r.float()).abs().max()):.3g}", flush=True)
    except Exception as e:  # noqa: BLE001
        first = e
        while first.__context__ is not None:
            first = first.__context__
        print(f"{name:32s} [{mode}] FAIL {type(first).__name__}: {str(first)[:160]}", flush=True)
        torch.cuda.synchronize()
        try:
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2):
                pass
        except Exception:  # noqa: BLE001
            pass


probe("torch.mm", lambda: a @ b)
probe("rms_norm_fwd", lambda: C.rms_norm_fwd(a, None, w, None, 1e-5))
probe("gemm 1cta (M=64)", lambda: C.gemm(a[:64].contiguous(), b))
probe("gemm (M=512)", lambda: C.gemm(a, b))
probe("gemm thread_local", lambda: C.gemm(a, b), "thread_local")
probe("gemm relaxed", lambda: C.gemm(a, b), "relaxed")
probe("swiglu_fwd", lambda: C.swiglu_fwd(a, a.clone()))
q = torch.randn(1, 512, 8, 128, device=dev, dtype=bf)
probe("attention_fwd", lambda: C.attention_fwd(q, q, q, 0.088, True))
probe("paddle.matmul", lambda: paddle.matmul(a.as_subclass(paddle.Tensor), b.as_subclass(paddle.Tensor)))

# ---- torch-side pieces of a ResNet / AMP step -------------------------------------------------------------------------------
import torch.nn.functional as TF  # noqa: E402

x4 = torch.randn(8, 64, 56, 56, device=dev, dtype=bf)
wc = torch.randn(64, 64, 3, 3, device=dev, dtype=bf)
probe("torch conv2d bf16", lambda: TF.conv2d(x4, wc, padding=1))
rm, rv = torch.zeros(64, device=dev), torch.ones(64, device=dev)
probe("torch batch_norm train", lambda: TF.batch_norm(x4, rm, rv, torch.ones(64, device=dev), torch.zeros(64, device=dev), True))
bn = paddle.nn.BatchNorm2D(64)
bn.to("gpu")
probe("paddle BatchNorm2D train", lambda: bn(x4.float().as_subclass(paddle.Tensor)))
conv = paddle.nn.Conv2D(64, 64, 3, padding=1)
conv.to("gpu")
probe("paddle Conv2D fp32", lambda: conv(x4.float().as_subclass(paddle.Tensor)))


def amp_conv():
    with paddle.amp.auto_cast(level="O2", dtype="bfloat16"):
        return conv(x4.as_subclass(paddle.Tensor))


probe("paddle Conv2D under auto_cast O2", amp_conv)
net = paddle.vision.models.resnet18(num_classes=10)
net.to("gpu")
xin = torch.randn(4, 3, 64, 64, device=dev).as_subclass(paddle.Tensor)


def fwd_nograd():
    with paddle.no_grad():
        return net(xin)


probe("resnet18 fwd no_grad fp32", fwd_nograd)


def fwd_bwd():
    for p in net.parameters():
        p.clear_grad()
    y = net(xin).sum()
    y.backward()
    return y.detach()


probe("resnet18 fwd+bwd fp32", fwd_bwd)
probe("resnet18 fwd+bwd thread_local", fwd_bwd, "thread_local")
qkv = torch.randn(1, 512, 3 * 8 * 128, device=dev, dtype=bf, requires_grad=True)
from paddle_b200.kernels import attention as KA  # noqa: E402


def attn_fb():
    qkv.grad = None
    o = KA.attention_packed(qkv.as_subclass(paddle.Tensor), 8, 8, causal=True)
    o.sum().backward()
    return qkv.grad.detach()


probe("attention packed fwd+bwd", attn_fb)
