"""The attention backward's dK/dV kernel, with and without its dQ stage, keeps its accumulators in registers and its wgmma pipelined:
read `cuobjdump -sass` of the built object and check every instantiation of attn_bwd::dkv_kernel for local-memory traffic (register
spills) and for fewer warpgroup-arrive fences than MMAs (a kernel that runs out of registers gets its wgmma serialized, warning C7512:
one WARPGROUP.ARRIVE per MMA)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "paddle_b200", "_build_cache", "attention_bwd_sm100.cuda.o")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(OBJ), reason="cuobjdump or the built object is missing")


def _dkv_kernels():
    out = subprocess.run(["cuobjdump", "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1) if "8attn_bwd10dkv_kernel" in m.group(1) else None
            if name:
                res[name] = {"mma": 0, "arrive": 0, "local": 0}
        elif name is not None:
            if re.search(r"\bHGMMA\.", line):
                res[name]["mma"] += 1
            elif "WARPGROUP.ARRIVE" in line:
                res[name]["arrive"] += 1
            elif re.search(r"\b(STL|LDL)\b", line):
                res[name]["local"] += 1
    return res


def test_dkv_kernel_instantiations_are_present():
    names = list(_dkv_kernels())
    # bf16 / fp16 x column mask or not x dQ stage or not
    assert len(names) == 8, names
    for stage in ("Lb0EEEv", "Lb1EEEv"):
        assert sum(stage in n for n in names) == 4, names


def test_dkv_kernel_does_not_spill():
    for k, v in _dkv_kernels().items():
        assert v["local"] == 0, (k, v)


def test_dkv_kernel_wgmma_is_pipelined():
    for k, v in _dkv_kernels().items():
        assert v["mma"] > 0, (k, v)
        assert v["arrive"] < v["mma"], (k, v)
