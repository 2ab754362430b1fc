"""The head_dim 64 training attention kernels, read from the built objects with `cuobjdump -sass`: attention_d64_sm100.cuda.o holds
exactly the dense / column-masked forward and the backward's dK/dV (with and without its dQ stage), dQ and stats kernels at D = 64, none
touches local memory and every wgmma kernel keeps its MMAs pipelined (fewer warpgroup-arrive fences than MMAs); and the head_dim 128
backward compiles to the instructions it compiled to before its bodies became templates on the head size
(tests/golden/attention_bwd_d128_sass.json: SHA-256 of each kernel's instructions, recorded before the change)."""
import json
import os
import re
import shutil
import subprocess

import pytest

from test_paged_attention_sass_cpu import sass_digests

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D64_OBJ = os.path.join(ROOT, "paddle_b200", "_build_cache", "attention_d64_sm100.cuda.o")
BWD_OBJ = os.path.join(ROOT, "paddle_b200", "_build_cache", "attention_bwd_sm100.cuda.o")
GOLDEN = os.path.join(ROOT, "tests", "golden", "attention_bwd_d128_sass.json")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None
                                or not all(os.path.exists(o) for o in (D64_OBJ, BWD_OBJ)), reason="cuobjdump, cu++filt or the built objects are missing")

DTYPES = ("__nv_bfloat16", "__half")
B = ("(bool)0", "(bool)1")


def _counts(obj):
    """{demangled kernel name: {"mma", "arrive", "local"}} over the object."""
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    res = {}
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = f.split("\n", 1)
        res[name.strip()] = {"mma": len(re.findall(r"\bHGMMA\.", body)), "arrive": body.count("WARPGROUP.ARRIVE"),
                             "local": len(re.findall(r"\b(?:STL|LDL)\b", body))}
    names = list(res)
    demangled = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return {d.strip(): res[n] for n, d in zip(names, demangled)}


def _expected():
    """Kernel name prefixes (up to the parameter list) of every D = 64 instantiation."""
    out = set()
    for t in DTYPES:
        for m in B:
            out.add(f"void b200::attn::fwd_kernel<{t}, {m}, (bool)0, {t}, (int)64>")
            out.add(f"void b200::attn_bwd::dq_d64_kernel<{t}, {m}>")
            out.add(f"void b200::attn_bwd::prep_d64_kernel<{t}, {m}>")         # ZERO_DQ (single pass) or not
            for dq in B:
                out.add(f"void b200::attn_bwd::dkv_d64_kernel<{t}, {m}, {dq}>")
    return out


def test_d64_object_holds_exactly_the_training_kernels():
    names = {n[:n.index(">(") + 1] for n in _counts(D64_OBJ)}
    assert names == _expected(), sorted(names ^ _expected())


def test_d64_kernels_use_no_local_memory():
    for n, c in _counts(D64_OBJ).items():
        assert c["local"] == 0, (n, c)


def test_d64_wgmma_kernels_are_pipelined():
    wgmma = {n: c for n, c in _counts(D64_OBJ).items() if "prep_d64_kernel" not in n}
    assert len(wgmma) == 16, sorted(wgmma)
    for n, c in wgmma.items():
        assert c["mma"] > 0 and c["arrive"] < c["mma"], (n, c)


def test_d128_backward_compiles_as_recorded():
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert sass_digests([BWD_OBJ]) == golden
