"""The tensor-core kernels keep their wgmma pipelined: read `cuobjdump -sass` of the built objects and check that every kernel issuing
warpgroup MMAs opens fewer warpgroup-arrive fences than it has MMAs. A function call anywhere in such a kernel (a device printf, a
__noinline__ helper) makes ptxas serialize every wgmma.mma_async (warning C7510): each MMA then gets its own WARPGROUP.ARRIVE and waits
for the previous one to retire."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CACHE = os.path.join(ROOT, "paddle_b200", "_build_cache")
KERNELS = {
    "gemm_sm100.cuda.o": "gemm_kernel",
    "gemm_fp8_sm100.cuda.o": "gemm_fp8_kernel",
    "gemm_wo_sm100.cuda.o": "wo_gemm_kernel",
    "attention_sm100.cuda.o": "4attn10fwd_kernel",
    "attention_bwd_sm100.cuda.o": "8attn_bwd9dq_kernel",
}
# not checked: 8attn_bwd10dkv_kernel, whose register spills and serialized MMAs are a separate change
# not checked: the MX (block-scaled) fp8 instantiations issue one MMA per 32-wide k-block and retire it before scaling, by design
EXCLUDE = re.compile(r"gemm_fp8_kernelILi\d+ELb[01]ELb[01]ELb1E")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not all(os.path.exists(os.path.join(CACHE, o)) for o in KERNELS),
                                reason="cuobjdump or the built objects are missing")


def _counts(obj):
    out = subprocess.run(["cuobjdump", "-sass", os.path.join(CACHE, obj)], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            res[name] = {"mma": 0, "arrive": 0}
        elif name is not None:
            if re.search(r"\b[HQI]GMMA\.", line):       # HGMMA bf16 / fp16, QGMMA fp8, IGMMA int8
                res[name]["mma"] += 1
            elif "WARPGROUP.ARRIVE" in line:
                res[name]["arrive"] += 1
    return res


@pytest.mark.parametrize("obj", sorted(KERNELS))
def test_wgmma_kernels_are_not_serialized(obj):
    use = {k: v for k, v in _counts(obj).items() if KERNELS[obj] in k and not EXCLUDE.search(k)}
    assert use, (obj, KERNELS[obj])
    for k, v in use.items():
        assert v["mma"] > 0, (k, v)
        assert v["arrive"] < v["mma"], (k, v)
