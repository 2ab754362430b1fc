"""Every kernel of the weight-only GEMM object compiles to the instructions recorded in tests/golden/wo_gemm_sass.json (digests as in
test_paged_attention_sass_cpu), and none uses local memory.  The golden file was recorded when the MoE expert GEMM was still a kernel of
its own (`wo_expert_gemm_kernel`, taking `ExpertParams`); it is now the EXPERTS = true instantiation of `wo_gemm_kernel`, whose dense
instantiations gained a `(bool)0` argument.  RENAMED maps the recorded names onto the current ones; the object must hold exactly the
mapped set of kernels, each with its recorded digest."""
import json
import os
import re
import shutil
import subprocess

import pytest

from test_paged_attention_sass_cpu import sass_digests

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ = os.path.join(ROOT, "paddle_b200", "_build_cache", "gemm_wo_sm100.cuda.o")
GOLDEN = os.path.join(ROOT, "tests", "golden", "wo_gemm_sass.json")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None or not os.path.exists(OBJ),
                                reason="cuobjdump, cu++filt or the built object is missing")

_ARGS = "(CUtensorMap_st, CUtensorMap_st, b200::wo::{})"


def _renamed():
    """{name when recorded: current name} of the 48 GEMM instantiations: token tile x int8 / int4 x bf16 / fp16 x scale group, dense and
    experts."""
    out = {}
    for ntok, wst in ((16, 8), (64, 4)):
        for int4 in (0, 1):
            for bf16 in (0, 1):
                for gs in (0, 64, 128):
                    t = f"<(int){ntok}, (int){wst}, (bool){int4}, (bool){bf16}, (int){gs}"
                    out[f"void b200::wo::wo_gemm_kernel{t}>{_ARGS.format('Params')}"] = f"void b200::wo::wo_gemm_kernel{t}, (bool)0>{_ARGS.format('Params')}"
                    out[f"void b200::wo::wo_expert_gemm_kernel{t}>{_ARGS.format('ExpertParams')}"] = \
                        f"void b200::wo::wo_gemm_kernel{t}, (bool)1>{_ARGS.format('Params')}"
    return out


RENAMED = _renamed()


def test_wo_gemm_kernels_compile_as_recorded():
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert set(RENAMED) <= set(golden), sorted(set(RENAMED) - set(golden))
    expected = {RENAMED.get(n, n): d for n, d in golden.items()}
    assert len(expected) == 48 + 6                                   # the GEMM instantiations and 2 formats x 3 outputs of wo_dequant_kernel
    assert sass_digests([OBJ]) == expected


def test_wo_gemm_kernels_use_no_local_memory():
    sass = subprocess.run(["cuobjdump", "-sass", OBJ], capture_output=True, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)[1:]
    assert len(funcs) == 48 + 6
    for f in funcs:
        name, body = f.split("\n", 1)
        assert not re.search(r"\b(LDL|STL)\b", body), name
