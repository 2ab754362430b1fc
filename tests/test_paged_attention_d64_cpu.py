"""The head_dim 64 attention kernels, read from the built objects with `cuobjdump -sass`: no d 64 instantiation touches local memory,
and every unwindowed head_dim 128 instantiation in attention_sm100.cu and decode_attention.cu compiles to the instructions it compiled
to before the head size became a template argument (tests/golden/attention_d128_sass.json: SHA-256 of each kernel's instructions, keyed
by its demangled name with the trailing head-size template argument, and the verify kernels' WINDOW = false after it, removed)."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJS = [os.path.join(ROOT, "paddle_b200", "_build_cache", f) for f in ("attention_sm100.cuda.o", "decode_attention.cuda.o")]
GOLDEN = os.path.join(ROOT, "tests", "golden", "attention_d128_sass.json")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None
                                or not all(os.path.exists(o) for o in OBJS), reason="cuobjdump, cu++filt or the built objects are missing")

HEAD = re.compile(r", \(int\)(64|128)(, \(bool\)0)?>\(")   # the head size as the last template argument of a kernel, or before WINDOW = false


def sass_functions(objs=OBJS):
    """{demangled kernel name: [instructions without their addresses]} over the objects."""
    out = {}
    for obj in objs:
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
        for f in re.split(r"\n\s*Function : ", sass)[1:]:
            name, body = f.split("\n", 1)
            out[name.strip()] = [re.sub(r"/\*[0-9a-f]{4}\*/", "", ln).strip() for ln in body.split("\n") if re.search(r"/\*[0-9a-f]{4}\*/", ln)]
    names = list(out)
    demangled = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return {d.strip(): out[n] for n, d in zip(names, demangled)}


def head_size(name):
    m = HEAD.search(name)
    return int(m.group(1)) if m else None


def windowed(name):
    """A sliding-window kernel (their instructions are checked by test_paged_attention_sass_cpu.py)."""
    return "_window_kernel" in name or ", (bool)1>(" in name


def d128_digests(funcs):
    """SHA-256 of every unwindowed kernel that is not a head_dim 64 instantiation, keyed by its name without the head-size argument."""
    return {HEAD.sub(">(", n): hashlib.sha256("\n".join(ins).encode()).hexdigest() for n, ins in funcs.items()
            if head_size(n) != 64 and not windowed(n)}


def test_unwindowed_d64_kernels_use_no_local_memory():
    d64 = {n: ins for n, ins in sass_functions().items() if head_size(n) == 64 and not windowed(n)}
    # decode split / merge, verify split / merge, paged prefill: bf16 and fp16 each
    kinds = ("decode_split_kernel", "decode_merge_kernel", "multi_split_kernel", "multi_merge_kernel", "fwd_kernel")
    assert sorted(sum(k + "<" in n for n in d64) for k in kinds) == [2] * len(kinds), sorted(d64)
    for n, ins in d64.items():
        assert not any(re.search(r"\b(LDL|STL)\b", i) for i in ins), n


def test_unwindowed_d128_kernels_compile_as_before():
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert d128_digests(sass_functions()) == golden
