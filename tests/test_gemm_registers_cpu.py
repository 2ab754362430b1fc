"""The GEMM's consumer warpgroups raise their register budget with `setmaxnreg.inc 224` and must actually get it: read
`cuobjdump -sass` of the built object and check that no `gemm_kernel` instantiation touches local memory and that every BN = 256
instantiation uses a register above R168, the most a thread can hold at the 384-thread launch budget.  ptxas sizes the whole kernel
at that budget when anything the consumers run can reach a trap (the bounded mbarrier wait), so this fails if one comes back."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "paddle_b200", "_build_cache", "gemm_sm100.cuda.o")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(OBJ),
                                reason="cuobjdump or the built object is missing")


def _scan():
    out = subprocess.run(["cuobjdump", "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    res, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            name = m.group(1)
            res[name] = {"max_reg": -1, "local": 0}
        elif name is not None:
            regs = [int(r) for r in re.findall(r"\bR(\d+)\b", line)]
            if regs:
                res[name]["max_reg"] = max(res[name]["max_reg"], max(regs))
            if re.search(r"\b(LDL|STL)\b", line):
                res[name]["local"] += 1
    return {k: v for k, v in res.items() if "gemm_kernel" in k}


def test_gemm_kernel_consumers_get_their_registers():
    kernels = _scan()
    assert kernels
    wide = {k: v for k, v in kernels.items() if "gemm_kernelILi256E" in k}
    assert len(wide) == 8, sorted(wide)
    for k, v in kernels.items():
        assert v["local"] == 0, (k, v)
    for k, v in wide.items():
        assert v["max_reg"] > 168, (k, v)
