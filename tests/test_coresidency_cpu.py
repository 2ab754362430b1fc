"""Resource numbers behind docs/race_detection.md ("cross-rank progress"): read `cuobjdump -res-usage` of the built objects and check the
statements the analysis relies on - the persistent GEMM fills an SM on its own, the peer-memory collectives are small,
bounded, non-persistent kernels that fit four to an SM."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CACHE = os.path.join(ROOT, "paddle_b200", "_build_cache")
SM_SMEM, SM_REGS, SM_THREADS, CTA_RESERVE = 228 * 1024, 65536, 2048, 1024

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(os.path.join(CACHE, "gemm_sm100.cuda.o")),
                                reason="cuobjdump or the built objects are missing")


def _usage(obj):
    out = subprocess.run(["cuobjdump", "-res-usage", os.path.join(CACHE, obj)], capture_output=True, text=True, check=True).stdout
    res = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:(\d+)", out):
        res[m.group(1)] = {"reg": int(m.group(2)), "stack": int(m.group(3)), "shared": int(m.group(4))}
    return res


def _const(src, name):
    text = open(os.path.join(ROOT, "paddle_b200", "csrc", src)).read()
    m = re.search(rf"constexpr\s+\w+\s+{name}\s*=\s*(\d+)\s*;", text)
    assert m, (src, name)
    return int(m.group(1))


def test_persistent_gemm_fills_the_sm():
    """One persistent GEMM CTA (3 warpgroups at the full launch register budget, most of the shared memory) leaves an SM no room for a
    CTA of the collectives: 512 threads need at least 512 x 16 registers.  The count is the allocation at launch, which
    `__launch_bounds__(384, 1)` fixes; `setmaxnreg` later moves registers between the CTA's warpgroups, not in or out of the CTA."""
    use = {k: v for k, v in _usage("gemm_sm100.cuda.o").items() if "gemm_kernel" in k}
    assert use
    threads = _const("gemm_sm100.cu", "kThreads")
    dyn = 4 * (128 * 64 * 2 + 256 * 64 * 2) + 1024 + 256       # Cfg<256>::SMEM_BYTES: four stages of the widest tile
    text = open(os.path.join(ROOT, "paddle_b200", "csrc", "gemm_sm100.cu")).read()
    assert "kStages = BN == 256 ? 4 : 6" in text and "kStages * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/" in text
    for k, v in use.items():
        assert v["reg"] * threads <= SM_REGS
        assert SM_REGS - v["reg"] * threads < 512 * 16, (k, v)  # the register file is the limiter: nothing co-resides
        assert dyn + v["shared"] + CTA_RESERVE <= SM_SMEM


def test_collective_kernels_are_small_and_pack_four_to_an_sm():
    use = {k: v for k, v in _usage("p2p_collectives.cuda.o").items() if any(n in k for n in ("allreduce", "reduce_scatter", "reduce_slots", "allgather", "alltoall", "a2av", "gather_pull"))}
    assert len(use) >= 8
    threads = _const("comm/p2p_collectives.cu", "kThreads")
    assert threads * 4 <= SM_THREADS
    for k, v in use.items():
        assert v["reg"] <= 128, (k, v)                         # 512 threads x 128 registers = one full register file at most
        assert v["reg"] * threads <= SM_REGS
        assert v["shared"] + CTA_RESERVE <= 4 * 1024, (k, v)   # a few hundred bytes of flags: never the limiter
    text = open(os.path.join(ROOT, "paddle_b200", "csrc", "comm", "p2p_collectives.cu")).read()
    grid_fn = text[text.index("static int comm_grid"):][:600]
    cap = int(re.search(r"const int cap = (\d+);", grid_fn).group(1))
    assert cap <= 132 // 2 and "while" not in grid_fn           # bounded grid (less than half the SMs), no persistent loop over a work queue
    # every device-side wait is bounded and traps
    assert text.count("__trap()") >= 1 and "10000000000" in text.replace("'", "").replace("ull", "")


def test_every_mbarrier_wait_in_the_tree_is_bounded():
    ptx = open(os.path.join(ROOT, "paddle_b200", "csrc", "include", "b200_ptx.cuh")).read()
    body = ptx[ptx.index("void mbar_wait("):][:1200]
    assert "__trap()" in body and "4000000000" in body
    for f in os.listdir(os.path.join(ROOT, "paddle_b200", "csrc")):
        if f.endswith(".cu"):
            src = open(os.path.join(ROOT, "paddle_b200", "csrc", f)).read()
            if "try_wait" in src:                                # a private wait loop must carry its own bound
                assert "__trap()" in src, f
