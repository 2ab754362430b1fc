"""KernelFactory: the table of kernels per (op, backend, dtype) and the selection rule.

Role parity: phi::KernelFactory / KernelKey / PD_REGISTER_KERNEL (paddle/phi/core/kernel_factory.h, kernel_registry.h) and the Python views
on it (`core._get_all_register_op_kernels`).  Here a kernel is a Python callable around a native launcher (or a reference composition); the
key is (backend, dtype) - layout is always dense row-major.  Selection: kernels registered for the op whose backend is the tensor's device
type (a custom-device plug-in registers under its own device type) and whose dtype set holds the tensor's dtype, highest priority first,
first one whose predicate accepts the arguments; an op with no kernel for a backend falls back to its `ANY` kernel (the ATen composition)."""
from __future__ import annotations

import importlib
from dataclasses import dataclass, field

import torch

HALF = ("float16", "bfloat16")
FLOAT = ("float16", "bfloat16", "float32")
ALL_FLOAT = FLOAT + ("float64",)


@dataclass(frozen=True)
class KernelKey:
    backend: str          # "GPU" | "CPU" | "ANY" | a custom device type
    dtype: str
    layout: str = "ANY"

    def __str__(self):
        return f"({self.backend}, {self.layout}, {self.dtype})"


@dataclass
class Kernel:
    op: str
    backend: str
    dtypes: tuple
    target: object                        # callable or "module:function" resolved on first use
    predicate: object = None              # (*args, **kwargs) -> bool
    native: str = ""                      # where the device code lives (csrc file :: launcher)
    priority: int = 0
    _fn: object = field(default=None, repr=False)

    @property
    def fn(self):
        if self._fn is None:
            t = self.target
            if isinstance(t, str):
                mod, name = t.split(":")
                t = getattr(importlib.import_module(mod if mod.startswith("paddle_b200") else "paddle_b200." + mod), name)
            self._fn = t
        return self._fn

    def keys(self):
        return [KernelKey(self.backend, d) for d in self.dtypes]

    def __call__(self, *args, **kwargs):
        return self.fn(*args, **kwargs)


def _is_keyed(a):
    """Arguments that carry a kernel key: torch tensors and plug-in device tensors (device.custom.CustomTensor: `.place`, numpy `.dtype`)."""
    return isinstance(a, torch.Tensor) or (hasattr(a, "place") and hasattr(a, "dtype") and hasattr(a.place, "get_device_type"))


def _dtype_name(t):
    return str(t.dtype).replace("torch.", "")


def _backend_of(t):
    if not isinstance(t, torch.Tensor):
        return t.place.get_device_type()                 # a custom device: its plug-in's device type is the backend
    if t.is_cuda:
        return "GPU"
    return "CPU"


class KernelFactory:
    _inst = None

    def __init__(self):
        self._table = {}
        self._builtin_loaded = False

    @classmethod
    def instance(cls):
        if cls._inst is None:
            cls._inst = KernelFactory()
        return cls._inst

    # ---- registration
    def register(self, op, backend, dtypes, target, predicate=None, native="", priority=0):
        k = Kernel(op, backend, tuple(dtypes), target, predicate, native, priority)
        lst = self._table.setdefault(op, [])
        lst.append(k)
        lst.sort(key=lambda e: -e.priority)
        return k

    def _ensure(self):
        if not self._builtin_loaded:
            self._builtin_loaded = True
            _register_builtin(self)

    # ---- queries
    def ops(self):
        self._ensure()
        return sorted(self._table)

    def kernels(self, op=None):
        self._ensure()
        if op is not None:
            return list(self._table.get(op, []))
        return {o: list(v) for o, v in self._table.items()}

    def has_kernel(self, op, key=None):
        self._ensure()
        ks = self._table.get(op, [])
        if key is None:
            return bool(ks)
        return any(k.backend == key.backend and key.dtype in k.dtypes for k in ks)

    def select(self, op, *args, **kwargs):
        """Kernel for this call (keyed by the first tensor argument)."""
        self._ensure()
        ks = self._table.get(op)
        if not ks:
            raise KeyError(f"no kernel is registered for op '{op}'")
        t = next((a for a in args if _is_keyed(a)), None)
        if t is None:
            t = next((a for a in kwargs.values() if _is_keyed(a)), None)
        if t is None:
            raise TypeError(f"op '{op}': kernel selection needs a tensor argument")
        backend, dt = _backend_of(t), _dtype_name(t)
        for want in (backend, "ANY"):
            for k in ks:
                if k.backend == want and (dt in k.dtypes or "*" in k.dtypes) and (k.predicate is None or k.predicate(*args, **kwargs)):
                    return k
        have = ", ".join(str(key) for k in ks for key in k.keys())
        raise NotImplementedError(f"op '{op}' has no kernel for {KernelKey(backend, dt)}; registered: {have}")

    def dispatch(self, op, *args, **kwargs):
        return self.select(op, *args, **kwargs)(*args, **kwargs)


def register_kernel(op, backend="GPU", dtypes=FLOAT, predicate=None, native="", priority=0):
    """Decorator form (PD_REGISTER_KERNEL): custom ops and device plug-ins add kernels to the same table."""
    def deco(fn):
        KernelFactory.instance().register(op, backend, dtypes, fn, predicate, native, priority)
        return fn

    return deco


def dispatch(op, *args, **kwargs):
    return KernelFactory.instance().dispatch(op, *args, **kwargs)


def all_registered_kernels():
    """{op: ["(backend, layout, dtype)", ...]} - the shape `core._get_all_register_op_kernels()` returns."""
    return {op: [str(key) for k in ks for key in k.keys()] for op, ks in KernelFactory.instance().kernels().items()}


# ---- the kernels of this package -------------------------------------------------------------------------------------------------------------
def _hd128(q, *a, **k):
    return q.shape[-1] == 128


def _register_builtin(f):
    G, A = "GPU", "ANY"
    r = f.register
    # GEMM family
    r("matmul", G, HALF, "kernels.gemm:matmul", native="csrc/gemm_sm100.cu::gemm_kernel, csrc/gemm_sm100.cu", priority=10)
    r("matmul", A, ("*",), "ops.linalg:matmul")
    r("linear", G, HALF, "kernels.gemm:linear", native="csrc/gemm_sm100.cu::gemm_kernel (bias / activation epilogues)", priority=10)
    r("linear", A, ("*",), "nn.functional:linear")
    r("fp8_gemm", G, ("float8_e4m3fn", "float8_e5m2"), "kernels.gemm_fp8:fp8_gemm", native="csrc/gemm_fp8_sm100.cu")
    r("fp8_quantize", G, FLOAT, "kernels.gemm_fp8:quantize_fp8", native="csrc/quant_fp8.cu")
    r("mx_quantize", G, FLOAT, "kernels.gemm_fp8:quantize_mx", native="csrc/quant_fp8.cu::mx_quantize_kernel")
    r("mx_gemm", G, ("float8_e4m3fn",), "kernels.gemm_fp8:mx_gemm", native="csrc/gemm_fp8_sm100.cu (MX scales applied in registers)")
    r("weight_only_linear", G, HALF, "nn.quant:weight_only_linear", native="csrc/gemm_wo_sm100.cu::wo_gemm_kernel", priority=10)
    r("weight_only_linear", A, ("*",), "nn.quant:weight_only_linear")
    # attention
    r("flash_attn", G, HALF, "kernels.attention:attention", predicate=_hd128, native="csrc/attention_sm100.cu, csrc/attention_bwd_sm100.cu", priority=10)
    r("flash_attn", A, ("*",), "kernels.attention:attention_ref")
    r("flash_attn_qkvpacked", G, HALF, "kernels.attention:attention_packed", native="csrc/attention_sm100.cu (packed qkv)")
    r("masked_multihead_attention", G, HALF, "incubate.nn.functional:masked_multihead_attention", native="csrc/decode_attention.cu")
    r("block_multihead_attention", G, HALF, "incubate.nn.paged_attention:block_attention", native="csrc/decode_attention.cu (paged), csrc/attention_sm100.cu (paged prefill), csrc/kv_cache_quant.cu (int8 / fp8 cache write)", priority=10)
    r("block_multihead_attention", A, ("*",), "incubate.nn.paged_attention:block_attention")
    # normalisation / activation / rotary / loss
    r("rms_norm", G, FLOAT, "kernels.norm:rms_norm", native="csrc/norm.cu::rms_norm_fwd / rms_norm_bwd", priority=10)
    r("rms_norm", A, ALL_FLOAT, "kernels.norm:rms_norm_ref")
    r("layer_norm", G, FLOAT, "kernels.norm:layer_norm", native="csrc/norm.cu::layer_norm_fwd / layer_norm_bwd", priority=10)
    r("layer_norm", A, ALL_FLOAT, "nn.functional:layer_norm")
    r("swiglu", G, FLOAT, "kernels.activation:swiglu", native="csrc/elementwise.cu::swiglu_fwd / swiglu_bwd", priority=10)
    r("swiglu", A, ALL_FLOAT, "incubate.nn.functional:swiglu")
    r("fused_rotary_position_embedding", G, FLOAT, "kernels.rope:apply_rope", native="csrc/elementwise.cu::rope_fwd", priority=10)
    r("fused_rotary_position_embedding", A, ALL_FLOAT, "kernels.rope:rope_ref")
    r("cross_entropy_with_softmax", G, FLOAT, "kernels.loss:softmax_cross_entropy", native="csrc/loss.cu::softmax_xent_fwd / bwd", priority=10)
    r("cross_entropy_with_softmax", A, ALL_FLOAT, "kernels.loss:softmax_cross_entropy")
    r("fused_bias_dropout_residual", G, FLOAT, "incubate.nn.functional:fused_dropout_add", native="csrc/fused_dropout.cu::bias_dropout_add_fwd")
    # MoE
    r("moe_expert_ffn", G, HALF, "kernels.moe:expert_ffn_grouped", native="csrc/moe.cu (routing), csrc/gemm_sm100.cu (grouped GEMM)")
    # fused blocks
    r("fused_rms_norm_linear", G, HALF, "kernels.fused_blocks:norm_linear", native="csrc/norm.cu + csrc/gemm_sm100.cu")
    r("fused_swiglu_linear", G, HALF, "kernels.fused_blocks:swiglu_linear", native="csrc/elementwise.cu + csrc/gemm_sm100.cu")
