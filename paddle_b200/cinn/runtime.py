"""Compile, cache and launch generated kernels.

A kernel is compiled once per (source, target): `nvcc -gencode arch=compute_90a,code=sm_90a` into a small shared object whose `extern "C"`
launcher is called through ctypes with raw device pointers and the current CUDA stream; the host target is `g++ -O2`.  Objects are cached
in-tree under `paddle_b200/_build_cache/cinn/` (keyed by the hash of the source), so a warm cache travels with the package.
Role parity: CINN's runtime module / NVRTC compile cache (paddle/cinn/runtime, paddle/cinn/backends/nvrtc)."""
from __future__ import annotations

import ctypes
import hashlib
import os
import shutil
import subprocess
import threading

import torch

from ..tensor import Tensor
from . import codegen

# in-tree by default (a warm cache travels with the package); B200_CINN_CACHE points it elsewhere (the test-suite uses a temporary directory)
_CACHE = os.environ.get("B200_CINN_CACHE") or os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "_build_cache", "cinn")
_LOCK = threading.Lock()
_LOADED = {}
_TORCH_DT = {"float32": torch.float32, "float64": torch.float64, "float16": torch.float16, "bfloat16": torch.bfloat16, "int32": torch.int32, "int64": torch.int64,
             "bool": torch.bool, "uint8": torch.uint8}

stats = {"compiled": 0, "cache_hits": 0, "launches": 0}


class CompileError(RuntimeError):
    pass


def _nvcc():
    return shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)


def compile_source(src, target, keep_source=True):
    """-> path of the shared object."""
    tag = hashlib.sha1((target + "\0" + src).encode()).hexdigest()[:20]
    os.makedirs(_CACHE, exist_ok=True)
    so = os.path.join(_CACHE, f"k_{target}_{tag}.so")
    if os.path.exists(so):
        stats["cache_hits"] += 1
        return so
    ext = "cu" if target == "cuda" else "cc"
    final_src = os.path.join(_CACHE, f"k_{target}_{tag}.{ext}")
    uniq = f"{os.getpid()}_{threading.get_ident()}"
    path = os.path.join(_CACHE, f"k_{target}_{tag}.{uniq}.{ext}")       # per-process names: the ranks of a job compile the same kernel at once
    with open(path, "w") as f:
        f.write(src)
    tmp = so + f".tmp{uniq}"
    if target == "cuda":
        nvcc = _nvcc()
        if nvcc is None:
            raise CompileError("nvcc not found: generated CUDA kernels cannot be built")
        cmd = [nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "--cudart", "shared", "-shared", "-Xcompiler", "-fPIC", "-o", tmp, path]
    else:
        cmd = ["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-fno-math-errno", "-o", tmp, path]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise CompileError(f"{' '.join(cmd)}\n{r.stderr[-4000:]}")
    os.replace(tmp, so)
    stats["compiled"] += 1
    if keep_source:
        os.replace(path, final_src)
    else:
        os.remove(path)
    return so


def _load(so):
    with _LOCK:
        lib = _LOADED.get(so)
        if lib is None:
            lib = _LOADED[so] = ctypes.CDLL(so)
        return lib


def _numel(shape):
    n = 1
    for d in shape:
        n *= int(d)
    return n


class FusedKernel:
    """Callable for one fusion group: tensors in operand order -> result tensor(s) in result order."""

    def __init__(self, spec):
        self.spec = spec
        self._fn = {}
        self.sources = {}
        self.launches = 0

    def source(self, target):
        if target not in self.sources:
            self.sources[target] = codegen.cuda_source(self.spec) if target == "cuda" else codegen.host_source(self.spec)
        return self.sources[target]

    def build(self, target):
        if target not in self._fn:
            lib = _load(compile_source(self.source(target), target))
            if target == "cuda":
                fn = lib.cinn_launch
                fn.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p), ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_int]
            else:
                fn = lib.cinn_run
                fn.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.POINTER(ctypes.c_void_p), ctypes.c_longlong, ctypes.c_int]
            fn.restype = ctypes.c_int
            self._fn[target] = fn
        return self._fn[target]

    def __call__(self, *tensors, **_attrs):
        if torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad for t in tensors):
            outs = list(_FusedFn.apply(self, *[t.as_subclass(torch.Tensor) if type(t) is not torch.Tensor else t for t in tensors]))
        else:
            outs = self._run(tensors)
            outs = list(outs) if isinstance(outs, tuple) else [outs]
        res = [o.as_subclass(Tensor) for o in finish(self.spec, outs)]
        return res[0] if len(res) == 1 else tuple(res)

    # ---- backward: one more generated kernel (cinn/autodiff.py); the torch interpreter when a derivative rule is missing --------------------
    def _backward_kernel(self, need):
        key = tuple(bool(v) for v in need)
        if not hasattr(self, "_bwd"):
            self._bwd = {}
        if key not in self._bwd:
            from .autodiff import backward_spec
            from .expr import Unsupported

            try:
                bspec, plan = backward_spec(self.spec, key)
                bk = FusedKernel(bspec) if bspec is not None else None
                if bk is not None:
                    bk.source("cuda")
                self._bwd[key] = (bk, plan)
            except Unsupported as e:
                self._bwd[key] = (None, None)
                self.backward_fallback = str(e)
        return self._bwd[key]

    def backward(self, inputs, grad_outputs, need):
        """Gradients of the inputs (None where not needed)."""
        spec = self.spec
        gouts = []
        for g, n in zip(grad_outputs, spec.outputs):
            if g is None:
                g = torch.zeros(n.shape, dtype=_TORCH_DT[n.dtype], device=inputs[0].device)
            gouts.append(g.contiguous())
        bk, plan = self._backward_kernel(need)
        if plan is None:                                           # no generated backward: differentiate the reference evaluation
            from .interp import evaluate

            with torch.enable_grad():
                xs = [t.detach().requires_grad_(bool(nd) and t.is_floating_point()) for t, nd in zip(inputs, need)]
                outs = evaluate(spec, xs, finished=False)
                pairs = [(o, g) for o, g in zip(outs, gouts) if o.requires_grad]
                wrt = [x for x in xs if x.requires_grad]
                gs = torch.autograd.grad([o for o, _ in pairs], wrt, [g for _, g in pairs], allow_unused=True) if pairs and wrt else []
            it = iter(gs)
            return [next(it) if x.requires_grad else None for x in xs]
        res = []
        if bk is not None:
            operands = [inputs[i] if kind == "in" else gouts[i] for kind, i in plan.inputs]
            res = bk._run(operands)
            res = list(res) if isinstance(res, tuple) else [res]
            res = [r.as_subclass(torch.Tensor) for r in res]
        grads = []
        for k, (t, nd) in enumerate(zip(inputs, need)):
            if not nd or k not in plan.parts:
                grads.append(None)
                continue
            acc = None
            seen = spec.inputs[k].shape                       # the shape the group read this tensor under (differs from t.shape for a view)
            for kind, i in plan.parts[k]:
                p = res[i] if kind == "out" else gouts[i]
                if tuple(p.shape) != tuple(seen):
                    p = p.sum_to_size(seen) if p.dim() >= len(seen) else p.reshape(seen)
                acc = p if acc is None else acc + p
            grads.append(None if acc is None else acc.reshape(t.shape).to(t.dtype))
        return grads

    def _run(self, tensors):
        spec = self.spec
        if len(tensors) != len(spec.inputs):
            raise TypeError(f"{spec.name}: expected {len(spec.inputs)} tensors, got {len(tensors)}")
        raw = []
        for t, n in zip(tensors, spec.inputs):
            t = t.as_subclass(torch.Tensor) if type(t) is not torch.Tensor else t
            if n.attrs.get("view") and tuple(t.shape) != n.shape and t.numel() == _numel(n.shape):
                t = t.contiguous().reshape(n.shape)                 # the group reads this tensor under another shape (per-channel statistics)
            if tuple(t.shape) != n.shape or t.dtype != _TORCH_DT[n.dtype]:
                raise TypeError(f"{spec.name}: operand is {list(t.shape)} {t.dtype}, the kernel was generated for {list(n.shape)} {n.dtype}")
            raw.append(t.detach().contiguous())
        dev = raw[0].device if raw else torch.device("cpu")
        if any(t.device != dev for t in raw):
            raise TypeError(f"{spec.name}: operands live on different devices")
        target = "cuda" if dev.type == "cuda" else "host"
        try:
            fn = self.build(target)
        except CompileError as e:
            # no compiler on this machine (or a build failure): the group still runs, through the reference evaluator - slow but correct
            if not getattr(self, "_warned", False):
                import warnings

                warnings.warn(f"paddle_b200.cinn: {spec.name} could not be built for {target}; running its reference evaluation instead\n{str(e)[:500]}")
                self._warned = True
            from .interp import evaluate

            with torch.no_grad():
                outs = evaluate(spec, raw, finished=False)
            res = [o.contiguous().as_subclass(Tensor) for o in outs]
            return res[0] if len(res) == 1 else tuple(res)
        outs = [torch.empty(n.shape, dtype=_TORCH_DT[n.dtype], device=dev) for n in spec.outputs]
        aux, scratch = 0, []
        if spec.col and target == "cuda":                       # partial sums of the column reductions: [split, A, B] per reduction
            aux = codegen.col_split(spec, torch.cuda.get_device_properties(dev).multi_processor_count)
            A, _, B = spec.akb
            scratch = [torch.empty(aux * A * B, dtype=torch.float64 if r.dtype == "float64" else torch.float32, device=dev) for r in spec.col]
        ins_p = (ctypes.c_void_p * max(len(raw), 1))(*[t.data_ptr() for t in raw])
        outs_p = (ctypes.c_void_p * (len(outs) + len(scratch)))(*[t.data_ptr() for t in outs + scratch])
        if target == "cuda":
            with torch.cuda.device(dev):
                aligned = all(t.data_ptr() % 16 == 0 for t in raw + outs)
                rc = fn(ins_p, outs_p, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream), int(aligned), spec.rows, aux)
            if rc != 0:
                raise RuntimeError(f"{spec.name}: kernel launch failed with CUDA error {rc}")
        else:
            rc = fn(ins_p, outs_p, spec.rows, 0)
            if rc != 0:
                raise RuntimeError(f"{spec.name}: host kernel returned {rc}")
        self.launches += 1
        stats["launches"] += 1
        res = [o.as_subclass(Tensor) for o in outs]
        return res[0] if len(res) == 1 else tuple(res)


def finish(spec, outs):
    """Results that are reductions to a scalar leave the kernel as per-row partials; the last step is one small library reduction."""
    res = []
    for o, n in zip(outs, spec.outputs):
        post = n.attrs.get("post")
        if post:
            o = o.as_subclass(torch.Tensor)
            o = {"sum": o.sum, "max": o.amax, "min": o.amin}[post]()
            if n.attrs.get("scale") is not None:
                o = o * n.attrs["scale"]
        res.append(o)
    return res


class _FusedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, kernel, *tensors):
        with torch.no_grad():
            outs = kernel._run(tensors)
        outs = tuple(o.as_subclass(torch.Tensor) for o in (outs if isinstance(outs, tuple) else (outs,)))
        ctx.kernel = kernel
        ctx.save_for_backward(*tensors)
        ctx.mark_non_differentiable(*[o for o in outs if not o.is_floating_point()])
        return outs

    @staticmethod
    def backward(ctx, *grad_outputs):
        grads = ctx.kernel.backward(list(ctx.saved_tensors), list(grad_outputs), ctx.needs_input_grad[1:])
        return (None, *grads)


def clear_cache():
    if os.path.isdir(_CACHE):
        shutil.rmtree(_CACHE)
    _LOADED.clear()
