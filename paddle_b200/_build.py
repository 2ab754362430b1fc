"""In-tree build + load of the native extension (``paddle_b200/_C*.so``).

* ``build()`` compiles every ``csrc/**/*.cu|cpp`` for sm_90a with ninja (cross-compiles without a GPU) into
  ``paddle_b200/_build_cache/`` and copies the module next to this file.
* ``load()`` imports the prebuilt module; on a GPU box a missing module is a hard error (no silent fallback).
"""
from __future__ import annotations

import glob
import importlib.util
import os
import shutil
import sys
import sysconfig

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(_HERE, "csrc")
_NAME = "_C"
_module = None

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "--expt-relaxed-constexpr", "-Xptxas", "-v", "--threads", "4",
]


def sources():
    srcs = sorted(glob.glob(os.path.join(_CSRC, "*.cu")) + glob.glob(os.path.join(_CSRC, "*.cpp"))
                  + glob.glob(os.path.join(_CSRC, "*", "*.cu")) + glob.glob(os.path.join(_CSRC, "*", "*.cpp")))
    return srcs


def so_path():
    suffix = sysconfig.get_config_var("EXT_SUFFIX") or ".so"
    return os.path.join(_HERE, _NAME + suffix)


def build(verbose: bool = False):
    """Compile the extension in-tree. Returns the path of the built shared object."""
    from torch.utils import cpp_extension

    from . import _wgmma_gen

    _wgmma_gen.main()
    build_dir = os.path.join(_HERE, "_build_cache")
    os.makedirs(build_dir, exist_ok=True)
    os.environ.setdefault("MAX_JOBS", str(os.cpu_count() or 8))
    mod = cpp_extension.load(
        name=_NAME,
        sources=sources(),
        extra_cflags=["-O3", "-std=c++17"],
        extra_cuda_cflags=NVCC_FLAGS,
        extra_include_paths=[_CSRC],
        build_directory=build_dir,
        with_cuda=True,
        verbose=verbose,
        is_python_module=True,
    )
    built = os.path.join(build_dir, _NAME + ".so")
    if os.path.exists(built):
        shutil.copy2(built, so_path())
    global _module
    _module = mod
    return so_path()


def load(required: bool = False):
    """Import the prebuilt extension. Returns None when it is absent (CPU-only dev box without a build)."""
    global _module
    if _module is not None:
        return _module
    path = so_path()
    if not os.path.exists(path):
        alt = os.path.join(_HERE, "_build_cache", _NAME + ".so")
        path = alt if os.path.exists(alt) else path
    if not os.path.exists(path):
        if required:
            raise RuntimeError(
                "paddle_b200 native extension is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                f"(expected {so_path()})")
        return None
    import torch  # noqa: F401  (libtorch must be loaded first)

    spec = importlib.util.spec_from_file_location(_NAME, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    sys.modules.setdefault("paddle_b200._C", mod)
    _module = mod
    return mod


def ext():
    """The extension, or raise if a CUDA tensor reaches a fused op without it."""
    m = load()
    if m is None:
        raise RuntimeError("paddle_b200: CUDA kernels requested but the native extension is missing (build it first)")
    return m
