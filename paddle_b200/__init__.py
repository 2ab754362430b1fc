"""paddle_b200 — a Blackwell(B200)-native deep-learning framework with the PaddlePaddle API surface.

``import paddle_b200 as paddle`` gives the reference's public namespace (python/paddle/__init__.py): Tensor, ops,
nn, optimizer, amp, io, jit, distributed (+fleet), vision, ... backed by PyTorch tensors/autograd for the plumbing
and hand-written sm_90a CUDA kernels (``paddle_b200/csrc``) for the hot paths.
"""
from __future__ import annotations

__version__ = "3.0.0"   # API level (see version.py); paddle_b200.version.b200_version is the framework's own version

import torch as _torch

from .framework import dtype as _dtype_mod
from .framework.dtype import (bfloat16, bool, complex64, complex128, dtype, finfo, float8_e4m3fn, float8_e5m2,  # noqa: A004,F401
                              float16, float32, float64, get_default_dtype, iinfo, int8, int16, int32, int64,
                              set_default_dtype, uint8)
from .framework.flags import get_flags, set_flags  # noqa: F401
from .framework.place import (CPUPlace, CUDAPinnedPlace, CUDAPlace, Place, get_device, is_compiled_with_cinn,  # noqa: F401
                              is_compiled_with_cuda, is_compiled_with_custom_device, is_compiled_with_distribute,
                              is_compiled_with_rocm, is_compiled_with_xpu, set_device)
from .framework.random import get_cuda_rng_state, get_rng_state, seed, set_cuda_rng_state, set_rng_state  # noqa: F401
from .tensor import Parameter, Tensor, is_tensor, to_tensor  # noqa: F401
from . import ops as _ops
from .ops import *  # noqa: F401,F403
from .ops import linalg as _linalg_ops  # noqa: F401
from . import autograd  # noqa: F401
from .autograd import PyLayer, enable_grad, grad, is_grad_enabled, no_grad, set_grad_enabled  # noqa: F401

half = float16
float = float32  # noqa: A001
double = float64
int = int32  # noqa: A001
long = int64

from . import nn, optimizer, amp, io, regularizer  # noqa: E402,F401
from .nn.layer import ParamAttr  # noqa: E402,F401
from .framework.io import async_save, clear_async_save_task_queue, load, save  # noqa: E402,F401
from . import distributed  # noqa: E402,F401
from . import kernels  # noqa: E402,F401


def __getattr__(name):
    """Lazy sub-packages (keeps `import paddle_b200` fast)."""
    import importlib

    lazy = {"vision", "metric", "hapi", "distribution", "sparse", "incubate", "jit", "static", "inference", "profiler", "quantization",
            "device", "text", "audio", "geometric", "models", "parallel", "utils", "fft", "signal", "linalg", "hub", "onnx", "callbacks",
            "sysconfig", "version", "base", "tensor_ns", "decomposition", "cost_model", "reader", "dataset", "tensorrt", "pir", "cinn", "_C_ops"}
    if name in lazy:
        return importlib.import_module("." + name, __name__)
    if name == "DataParallel":
        from .distributed.data_parallel import DataParallel

        return DataParallel
    if name in ("Model", "summary", "flops"):
        from . import hapi

        return getattr(hapi, name)
    if name == "batch":
        from .reader import batch

        return batch
    if name in ("disable_static", "enable_static", "in_dynamic_mode"):
        from . import static

        return getattr(static, name)
    if name in ("set_grad_enabled",):
        from .autograd import set_grad_enabled

        return set_grad_enabled
    if name in ("get_cuda_rng_state",):
        from .framework import random

        return getattr(random, name)
    raise AttributeError(f"module 'paddle_b200' has no attribute '{name}'")


def install_as_paddle():
    """Register this package under the name ``paddle`` so reference user code runs unchanged."""
    import sys

    sys.modules.setdefault("paddle", sys.modules[__name__])
    for k, v in list(sys.modules.items()):
        if k.startswith(__name__ + "."):
            sys.modules.setdefault("paddle" + k[len(__name__):], v)


from . import _compat_paths as _compat_paths  # noqa: E402

from .framework import flags as _flags_mod  # noqa: E402

if _flags_mod.flag("FLAGS_b200_native_allocator", False):      # before anything touches the GPU
    from .device.cuda import use_auto_growth_allocator as _use_native_allocator

    _use_native_allocator()
_compat_paths.install()
