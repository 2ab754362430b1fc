"""Python face of the sm_90a kernels (csrc/).  Each op is a torch.autograd.Function around the native launchers;
CPU tensors take a plain-PyTorch reference path (used by the CPU test-suite), CUDA tensors REQUIRE the extension."""
from __future__ import annotations

import torch

from .._build import ext, load
from ..framework.flags import flag


def use_fused(t: torch.Tensor) -> bool:
    return t.is_cuda and flag("FLAGS_use_fused_kernels", True)


def launch_count() -> int:
    m = load()
    return int(m.launch_count()) if m is not None else 0


def reset_launch_count():
    m = load()
    if m is not None:
        m.reset_launch_count()


def raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


def wrap(t):
    from ..tensor import Tensor

    if isinstance(t, torch.Tensor) and not isinstance(t, Tensor):
        return t.as_subclass(Tensor)
    return t
