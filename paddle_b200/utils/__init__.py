"""paddle.utils. Parity: python/paddle/utils/__init__.py."""
from __future__ import annotations

import functools
import importlib
import warnings

from ..framework import unique_name  # noqa: F401
from . import cpp_extension, dlpack, download  # noqa: F401


def deprecated(update_to="", since="", reason="", level=0):
    def deco(fn):
        @functools.wraps(fn)
        def wrapper(*a, **k):
            msg = f"API '{fn.__module__}.{fn.__name__}' is deprecated since {since}" + (f", use '{update_to}' instead" if update_to else "") + (f". {reason}" if reason else "")
            if level >= 2:
                raise RuntimeError(msg)
            if level == 1 or level == 0:
                warnings.warn(msg, category=DeprecationWarning, stacklevel=2)
            return fn(*a, **k)

        return wrapper

    return deco


def try_import(module_name, err_msg=None):
    try:
        return importlib.import_module(module_name)
    except ImportError as e:
        raise ImportError(err_msg or f"Failed importing {module_name}. This likely means that some paddle modules require additional dependencies.") from e


def require_version(min_version, max_version=None):
    from .. import __version__

    def key(v):
        return tuple(int(x) for x in str(v).split(".")[:3] if x.isdigit())

    cur = key(__version__)
    if cur == (0, 0, 0):   # development build: every requirement is accepted, as in the reference
        return
    if cur < key(min_version) or (max_version is not None and cur > key(max_version)):
        raise Exception(f"paddle version {__version__} does not satisfy the requirement [{min_version}, {max_version or 'inf'}]")


def run_check():
    """paddle.utils.run_check(): trains a tiny model on every visible device through the native kernels."""
    import torch

    from .. import nn, optimizer, randn, set_device

    devs = ["cpu"] + ([f"gpu:{i}" for i in range(torch.cuda.device_count())] if torch.cuda.is_available() else [])
    for d in devs[-1:]:
        set_device(d)
        m = nn.Linear(8, 8)
        o = optimizer.SGD(0.1, parameters=m.parameters())
        x = randn([4, 8])
        l = (m(x) ** 2).mean()
        l.backward()
        o.step()
        print(f"paddle_b200 works on {d}.")
    if torch.cuda.is_available():
        from .._build import load

        print("native sm_90a extension:", "loaded" if load() is not None else "NOT BUILT")
    print("PaddlePaddle-compatible paddle_b200 is installed successfully!")


def flops(op_type, input_shapes, attrs=None):
    """FLOPs of one operator from its input shapes. Parity: python/paddle/utils/flops.py:flops (per-op registry; unknown ops give 0).
    The model-level counter is `paddle.flops(net, input_size)`."""
    from functools import reduce
    from operator import mul

    attrs = attrs or {}

    def numel(shape):
        return reduce(mul, shape, 1)

    def first(key):
        v = input_shapes.get(key)
        return v[0] if v and isinstance(v[0], (list, tuple)) else v

    t = op_type
    if t in ("matmul", "matmul_v2"):
        x, y = list(first("X")), list(first("Y"))
        if attrs.get("transpose_X") or attrs.get("trans_x"):
            x[-1], x[-2] = x[-2], x[-1]
        if attrs.get("transpose_Y") or attrs.get("trans_y"):
            y[-1], y[-2] = y[-2], y[-1]
        batch = x[:-2] if len(x) >= len(y) else y[:-2]
        return 2 * numel(batch) * x[-2] * x[-1] * y[-1]
    if t in ("elementwise_add", "elementwise_sub", "elementwise_mul", "elementwise_div", "add", "subtract", "multiply", "divide"):
        x, y = first("X"), first("Y")
        return max(numel(x), numel(y))
    if t in ("relu", "gelu", "silu", "sigmoid", "tanh", "dropout", "softmax"):
        x = first("X")
        return numel(x) * (3 if t == "softmax" else 1)
    if t == "layer_norm":
        x = first("X")
        return numel(x) * (8 if attrs.get("epsilon") is not None else 7)
    if t in ("conv2d", "depthwise_conv2d"):
        x, w = first("Input"), first("Filter")
        stride, pad, dil = attrs.get("strides", [1, 1]), attrs.get("paddings", [0, 0]), attrs.get("dilations", [1, 1])
        ho = (x[2] + 2 * pad[0] - dil[0] * (w[2] - 1) - 1) // stride[0] + 1
        wo = (x[3] + 2 * pad[1] - dil[1] * (w[3] - 1) - 1) // stride[1] + 1
        return 2 * x[0] * w[0] * ho * wo * w[1] * w[2] * w[3]
    if t in ("reshape2", "transpose2", "slice", "concat", "split", "unsqueeze2", "squeeze2", "c_embedding", "lookup_table_v2"):
        return 0
    return 0


