"""Every kernel of the paged attention objects compiles to the instructions recorded in tests/golden/paged_attention_sass.json, read from
the built objects with `cuobjdump -sass`.  The golden file holds the SHA-256 of each kernel's instructions (addresses removed, runs of
blanks collapsed: cuobjdump pads its columns to the widest instruction in the object, so the same kernel in another object would hash
differently), keyed by its demangled name when it was recorded.  RENAMED maps the names that have changed since onto the current ones;
the objects must hold exactly the mapped set of kernels, each with its recorded digest."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJS = [os.path.join(ROOT, "paddle_b200", "_build_cache", f) for f in ("attention_sm100.cuda.o", "decode_attention.cuda.o")]
GOLDEN = os.path.join(ROOT, "tests", "golden", "paged_attention_sass.json")

pytestmark = pytest.mark.skipif(shutil.which("cuobjdump") is None or shutil.which("cu++filt") is None
                                or not all(os.path.exists(o) for o in OBJS), reason="cuobjdump, cu++filt or the built objects are missing")

_MERGE = "(const float *, const float *, T1 *, int)"
_SPLIT = "(const T1 *, const T1 *, const T1 *, const int *, float *, float *, int, int, int, int, float, const int *, int, int, int)"
_Q8 = ("(const T1 *, const unsigned char *, const unsigned char *, const int *, float *, float *, int, int, int, float, const float *, "
       "const float *, const int *, int, int, int)")
_FWD = ("(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, b200::attn::WindowParams<std::conditional<std::is_same<T2, T1>::value, "
        "b200::attn::PagedParams, b200::attn::QuantPagedParams>::type>)")
_MULTI = "(b200::decode_multi::Params)"


def _renamed():
    """{name when recorded: current name} of the kernels renamed when the sliding-window kernels moved next to their unwindowed
    siblings, the verify kernels took the head size and the window as template arguments, and the windowed decode and verify launches
    went to the unwindowed merge kernels (which compiled to the same instructions)."""
    out = {"b200::window::paged_work_window_kernel(const int *, const int *, int, int, int *, int2 *, int)":
           "b200::attn::paged_work_window_kernel(const int *, const int *, int, int, int *, int2 *, int)"}
    for t in ("__half", "__nv_bfloat16"):
        out[f"void b200::decode_multi::multi_merge_kernel<{t}>{_MULTI}"] = f"void b200::decode_multi::multi_merge_kernel<{t}, (int)128>{_MULTI}"
        out[f"void b200::decode_verify64::multi_merge_kernel<{t}>(b200::decode_verify64::Params)"] = \
            f"void b200::decode_multi::multi_merge_kernel<{t}, (int)64>{_MULTI}"
        out[f"void b200::decode_verify64::multi_split_kernel<{t}>(b200::decode_verify64::Params)"] = \
            f"void b200::decode_multi::multi_split_kernel<{t}, {t}, (int)64, (bool)0>{_MULTI}"
        for d in (128, 64):
            out[f"void b200::window::decode_split_window_kernel<{t}, (int){d}>{_SPLIT}"] = f"void b200::decode::decode_split_window_kernel<{t}, (int){d}>{_SPLIT}"
            out[f"void b200::window::decode_merge_window_kernel<{t}, (int){d}>{_MERGE}"] = f"void b200::decode::decode_merge_kernel<{t}, (int){d}>{_MERGE}"
            out[f"void b200::window::multi_merge_window_kernel<{t}, (int){d}>(b200::window::MultiParams)"] = \
                f"void b200::decode_multi::multi_merge_kernel<{t}, (int){d}>{_MULTI}"
        for kv in (t, "b200::kv8::I8", "b200::kv8::E4M3"):
            out[f"void b200::decode_multi::multi_split_kernel<{t}, {kv}>{_MULTI}"] = f"void b200::decode_multi::multi_split_kernel<{t}, {kv}, (int)128, (bool)0>{_MULTI}"
        for kv, d in ((t, 128), (t, 64), ("b200::kv8::I8", 128), ("b200::kv8::E4M3", 128)):
            out[f"void b200::window::multi_split_window_kernel<{t}, {kv}, (int){d}>(b200::window::MultiParams)"] = \
                f"void b200::decode_multi::multi_split_kernel<{t}, {kv}, (int){d}, (bool)1>{_MULTI}"
            out[f"void b200::window::fwd_window_kernel<{t}, {kv}, (int){d}>{_FWD}"] = f"void b200::attn::fwd_window_kernel<{t}, {kv}, (int){d}>{_FWD}"
        for kv in ("b200::kv8::I8", "b200::kv8::E4M3"):
            out[f"void b200::window::decode_split_q8_window_kernel<{t}, {kv}>{_Q8}"] = f"void b200::decode::decode_split_q8_window_kernel<{t}, {kv}>{_Q8}"
    return out


RENAMED = _renamed()


def sass_digests(objs=OBJS):
    """{demangled kernel name: SHA-256 of its instructions} over the objects."""
    out = {}
    for obj in objs:
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
        for f in re.split(r"\n\s*Function : ", sass)[1:]:
            name, body = f.split("\n", 1)
            ins = [" ".join(re.sub(r"/\*[0-9a-f]{4}\*/", "", ln).split()) for ln in body.split("\n") if re.search(r"/\*[0-9a-f]{4}\*/", ln)]
            out[name.strip()] = hashlib.sha256("\n".join(ins).encode()).hexdigest()
    names = list(out)
    demangled = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return {d.strip(): out[n] for n, d in zip(names, demangled)}


def test_paged_attention_kernels_compile_as_recorded():
    with open(GOLDEN) as f:
        golden = json.load(f)
    assert set(RENAMED) <= set(golden), sorted(set(RENAMED) - set(golden))
    expected = {}
    for n, d in golden.items():                                # kernels merged into one must have compiled to the same instructions
        assert expected.setdefault(RENAMED.get(n, n), d) == d, n
    assert sass_digests() == expected
