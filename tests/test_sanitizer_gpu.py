"""Automated compute-sanitizer pass (racecheck + memcheck) over the hand-written HBM-bound kernels on small shapes.
wgmma / TMA kernels are left out: the tools do not model the async proxy, and replay makes them take minutes (docs/race_detection.md)."""
import os
import shutil
import subprocess
import sys

import pytest
import torch

SANITIZER = shutil.which("compute-sanitizer") or ("/usr/local/cuda/bin/compute-sanitizer" if os.path.exists("/usr/local/cuda/bin/compute-sanitizer") else None)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORKLOAD = r"""
import torch
import paddle_b200 as paddle
from paddle_b200._build import ext
from paddle_b200.kernels import norm, activation as act
from paddle_b200.incubate.nn import functional as IF
E = ext()
torch.manual_seed(0)
P = lambda t: t.as_subclass(paddle.Tensor)
x = torch.randn(64, 1024, device="cuda", dtype=torch.bfloat16, requires_grad=True)
w = torch.randn(1024, device="cuda", dtype=torch.bfloat16, requires_grad=True)
norm.rms_norm(P(x), P(w), 1e-6).as_subclass(torch.Tensor).float().sum().backward()
norm.layer_norm(P(x), [1024], P(w), P(w), 1e-5).as_subclass(torch.Tensor).float().sum().backward()
g = torch.randn(64, 2048, device="cuda", dtype=torch.bfloat16, requires_grad=True)
act.swiglu(P(g)).as_subclass(torch.Tensor).float().sum().backward()
IF.fused_dropout_add(P(x.detach()), P(x.detach()), p=0.3, training=True)
IF.fused_bias_act(P(g.detach()), P(torch.zeros(2048, device="cuda", dtype=torch.bfloat16)), act_method="swiglu")
lin = paddle.nn.Linear(256, 256).to("cuda")
opt = paddle.optimizer.AdamW(1e-3, parameters=lin.parameters())
(lin(P(torch.randn(32, 256, device="cuda"))) ** 2).mean().backward()
opt.step()
logits = torch.randn(128, 4096, device="cuda", dtype=torch.bfloat16, requires_grad=True)
paddle.nn.functional.cross_entropy(P(logits), P(torch.randint(0, 4096, (128,), device="cuda"))).backward()
q, sf = E.quantize_mx(torch.randn(128, 256, device="cuda", dtype=torch.bfloat16))
E.dequantize_mx(q, sf)
torch.cuda.synchronize()
print("WORKLOAD_DONE")
"""


def _run(tool, extra=(), workload=WORKLOAD):
    cmd = [SANITIZER, "--tool", tool, "--error-exitcode", "17", *extra, sys.executable, "-c", workload]
    return subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=900)


PROBE = "import torch; torch.zeros(4, device='cuda').add_(1); torch.cuda.synchronize(); print('PROBE_DONE')"


@pytest.mark.gpu
@pytest.mark.skipif(SANITIZER is None, reason="compute-sanitizer is not installed")
@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_compute_sanitizer_clean(tool):
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    # a library-only process first.  Where the tool cannot attach to the driver, the first CUDA call of ANY process under it fails
    # with cudaErrorUnknown: that, and only that, is a reason to skip; a probe that fails in another way is a broken set-up
    probe = _run(tool, workload=PROBE)
    if "PROBE_DONE" not in probe.stdout:
        assert "cudaErrorUnknown" in probe.stdout + probe.stderr, (probe.stdout + probe.stderr)[-2000:]
        pytest.skip("compute-sanitizer cannot instrument CUDA processes here (cudaErrorUnknown under the tool in a torch-only process)")
    r = _run(tool, ("--racecheck-report", "all") if tool == "racecheck" else ())
    tail = (r.stdout + r.stderr)[-4000:]
    assert "WORKLOAD_DONE" in r.stdout, tail
    assert r.returncode == 0, tail
    if tool == "racecheck":
        assert "RACECHECK SUMMARY: 0 hazards displayed (0 errors, 0 warnings)" in r.stdout + r.stderr, tail
    else:
        assert "ERROR SUMMARY: 0 errors" in r.stdout + r.stderr, tail
