"""paddle.utils.cpp_extension: build custom C++/CUDA ops for sm_90a.
Parity: python/paddle/utils/cpp_extension/{cpp_extension,extension_utils}.py (load, setup, CppExtension, CUDAExtension).

Custom ops are pybind/torch extensions compiled with ``-gencode arch=compute_90a,code=sm_90a``; functions exported
from the module operate on paddle_b200 Tensors (they are torch tensors underneath)."""
from __future__ import annotations

import os

SM100_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--expt-relaxed-constexpr"]


def _wrap_module(mod):
    import torch

    from ..tensor import Tensor

    class _Wrapped:
        def __getattr__(self, name):
            fn = getattr(mod, name)
            if not callable(fn):
                return fn

            def call(*a, **k):
                out = fn(*[x.as_subclass(torch.Tensor) if isinstance(x, torch.Tensor) else x for x in a], **k)
                conv = lambda o: o.as_subclass(Tensor) if isinstance(o, torch.Tensor) else o  # noqa: E731
                return type(out)(conv(o) for o in out) if isinstance(out, (list, tuple)) else conv(out)

            return call

    return _Wrapped()


def load(name, sources, extra_cxx_cflags=None, extra_cuda_cflags=None, extra_ldflags=None, extra_include_paths=None, build_directory=None, verbose=False):
    from torch.utils import cpp_extension as ce

    build_directory = build_directory or os.path.join(os.path.expanduser("~"), ".cache", "paddle_b200_extensions", name)
    os.makedirs(build_directory, exist_ok=True)
    has_cuda = any(s.endswith((".cu", ".cuh")) for s in sources)
    mod = ce.load(name=name, sources=list(sources), extra_cflags=list(extra_cxx_cflags or []) + ["-O3", "-std=c++17"],
                  extra_cuda_cflags=SM100_FLAGS + list(extra_cuda_cflags or []), extra_ldflags=extra_ldflags, extra_include_paths=extra_include_paths,
                  build_directory=build_directory, with_cuda=has_cuda, verbose=verbose)
    return _wrap_module(mod)


def CppExtension(sources, *args, **kwargs):
    from torch.utils import cpp_extension as ce

    return ce.CppExtension(kwargs.pop("name", "custom_ops"), sources, *args, **kwargs)


def CUDAExtension(sources, *args, **kwargs):
    from torch.utils import cpp_extension as ce

    kwargs.setdefault("extra_compile_args", {"cxx": ["-O3", "-std=c++17"], "nvcc": SM100_FLAGS})
    return ce.CUDAExtension(kwargs.pop("name", "custom_ops"), sources, *args, **kwargs)


def setup(**attr):
    from setuptools import setup as _setup
    from torch.utils import cpp_extension as ce

    attr.setdefault("cmdclass", {})["build_ext"] = ce.BuildExtension
    if "ext_modules" in attr and not isinstance(attr["ext_modules"], (list, tuple)):
        attr["ext_modules"] = [attr["ext_modules"]]
    return _setup(**attr)


def get_build_directory(verbose=False):
    return os.path.join(os.path.expanduser("~"), ".cache", "paddle_b200_extensions")
