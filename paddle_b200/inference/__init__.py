"""paddle.inference. Parity: python/paddle/inference/wrapper.py, paddle/fluid/inference/api/analysis_predictor.cc
(Config, create_predictor, Predictor, Tensor handles, PrecisionType, PlaceType, get_version...).

The predictor loads ``jit.save`` artifacts (prefix.pdmodel + prefix.pdiparams) and serves them with CUDA-graph replay
per input signature (jit.StaticFunction) - the sm_90a answer to the reference's IR-pass + TensorRT pipeline."""
from __future__ import annotations

import enum
import os

import numpy as np
import torch

from ..tensor import to_tensor


class PrecisionType(enum.Enum):
    Float32 = 0
    Half = 1
    Int8 = 2
    Bfloat16 = 3


class PlaceType(enum.Enum):
    UNK = -1
    CPU = 0
    GPU = 1
    XPU = 2
    CUSTOM = 3


class DataType(enum.Enum):
    FLOAT32 = 0
    INT64 = 1
    INT32 = 2
    UINT8 = 3
    INT8 = 4
    FLOAT16 = 5
    BOOL = 6
    FLOAT64 = 7
    BFLOAT16 = 8


class Config:
    def __init__(self, model_dir_or_prog=None, params_file=None):
        self._prefix = None
        if model_dir_or_prog is not None:
            self.set_model(model_dir_or_prog, params_file)
        self._use_gpu, self._gpu_id, self._precision = False, 0, PrecisionType.Float32
        self._memory_optim, self._ir_optim, self._glog, self._threads = False, True, True, 1

    def set_model(self, prog_file, params_file=None):
        p = prog_file
        for suf in (".pdmodel", ".json"):
            if p.endswith(suf):
                p = p[: -len(suf)]
        self._prefix = p

    def set_prog_file(self, f):
        self.set_model(f)

    def set_params_file(self, f):
        pass

    def prog_file(self):
        return self._prefix + ".pdmodel"

    def params_file(self):
        return self._prefix + ".pdiparams"

    def model_dir(self):
        return os.path.dirname(self._prefix or "")

    def enable_use_gpu(self, memory_pool_init_size_mb=100, device_id=0, precision_mode=PrecisionType.Float32):
        self._use_gpu, self._gpu_id, self._precision = True, device_id, precision_mode

    def disable_gpu(self):
        self._use_gpu = False

    def use_gpu(self):
        return self._use_gpu

    def gpu_device_id(self):
        return self._gpu_id

    def enable_memory_optim(self, x=True):
        self._memory_optim = x

    def switch_ir_optim(self, x=True):
        self._ir_optim = x

    def ir_optim(self):
        return self._ir_optim

    def switch_use_feed_fetch_ops(self, x=False):
        pass

    def switch_specify_input_names(self, x=True):
        pass

    def set_cpu_math_library_num_threads(self, n):
        self._threads = n
        torch.set_num_threads(max(1, int(n)))

    def cpu_math_library_num_threads(self):
        return self._threads

    def enable_mkldnn(self):
        pass

    def disable_glog_info(self):
        self._glog = False

    def enable_tensorrt_engine(self, *a, **k):
        """TensorRT subgraphs are replaced by the native CUDA-graph path; accepted for config compatibility."""
        self._trt = True

    def tensorrt_engine_enabled(self):
        return getattr(self, "_trt", False)

    def set_trt_dynamic_shape_info(self, *a, **k):
        pass

    def enable_cuda_graph(self):
        self._cuda_graph = True

    def summary(self):
        return f"Config(prefix={self._prefix}, gpu={self._use_gpu}, precision={self._precision.name})"

    # ---- optimisation pipeline.  Parity: the analysis predictor's IR pass list (paddle/fluid/inference/api/paddle_pass_builder.cc).  For a
    # saved PROGRAM artifact (static.save_inference_model / a traced program) the pass names map onto the native IR passes of
    # paddle_b200.pir and are really run when the predictor is created (switch_ir_optim(False) or an empty list skips them); a pickled
    # Layer artifact executes through the hand-written kernels directly and the list is only recorded.
    _PASSES = ["conv_bn_fuse_pass", "identity_op_clean_pass", "common_subexpression_elimination_pass", "constant_folding_pass", "dead_code_elimination_pass", "fuse_gemm_epilogue_pass",
               "fused_swiglu_pass", "add_norm_fuse_pass", "inplace_pass"]
    _PASS_TO_PIR = {
        "conv_bn_fuse_pass": ["conv_bn_fuse"], "conv_eltwiseadd_bn_fuse_pass": ["conv_bn_fuse"], "identity_op_clean_pass": ["identity_elim"], "common_subexpression_elimination_pass": ["cse"], "constant_folding_pass": ["constant_fold"],
        "dead_code_elimination_pass": ["dce"], "fuse_gemm_epilogue_pass": ["fuse_matmul_add", "fuse_linear_act_gelu", "fuse_linear_act_relu"],
        "matmul_add_act_fuse_pass": ["fuse_matmul_add", "fuse_linear_act_gelu", "fuse_linear_act_relu"], "fused_swiglu_pass": ["fuse_swiglu"],
        "add_norm_fuse_pass": ["fuse_add_rms_norm"], "inplace_pass": ["inplace"],
        # the short names the round-1 list used
        "constant_folding": ["constant_fold"], "common_subexpression_elimination": ["cse"], "fuse_gemm_epilogue": ["fuse_matmul_add", "fuse_linear_act_gelu", "fuse_linear_act_relu"],
        "dead_code_elimination": ["dce"],
    }

    def _pir_passes(self):
        """The configured pass list as native pass names (dead code is swept before and after the fusions)."""
        if not getattr(self, "_ir_optim", True):
            return []
        out = []
        for name in self._opt()["passes"]:
            for p in self._PASS_TO_PIR.get(name, [name] if name in ("dce", "cse", "identity_elim", "constant_fold", "inplace", "conv_bn_fuse") else []):
                if p not in out or p == "dce":
                    out.append(p)
        if out and "dce" in out:
            first_fuse = next((i for i, p in enumerate(out) if p.startswith("fuse_")), None)
            if first_fuse is not None and "dce" not in out[:first_fuse]:
                out.insert(first_fuse, "dce")
            if not out[-1] in ("dce", "inplace"):
                out.append("dce")
        return out

    def _opt(self):
        return self.__dict__.setdefault("_options", {"passes": list(self._PASSES)})

    def pass_builder(self):
        cfg = self

        class _PassBuilder:
            def all_passes(self):
                return list(cfg._opt()["passes"])

            def append_pass(self, name):
                cfg._opt()["passes"].append(name)

            def insert_pass(self, idx, name):
                cfg._opt()["passes"].insert(idx, name)

            def delete_pass(self, name):
                cfg.delete_pass(name)

            def set_passes(self, passes):
                cfg._opt()["passes"] = list(passes)

            def turn_on_debug(self):
                cfg._opt()["ir_debug"] = True

        return _PassBuilder()

    def delete_pass(self, name):
        p = self._opt()["passes"]
        for cand in (name, name + "_pass", name[:-5] if name.endswith("_pass") else name):     # "constant_folding" == "constant_folding_pass"
            if cand in p:
                p.remove(cand)
                return

    def enable_custom_passes(self, passes, custom_pass_only=False):
        self._opt()["passes"] = (list(passes) if custom_pass_only else self._opt()["passes"] + list(passes))

    def switch_ir_debug(self, x=True, passes=None):
        self._opt()["ir_debug"] = bool(x)

    def set_optimization_level(self, level):
        self._opt()["opt_level"] = int(level)

    def set_optim_cache_dir(self, d):
        self._opt()["optim_cache_dir"] = d

    def enable_save_optim_model(self, flag=True):
        self._opt()["save_optim_model"] = bool(flag)

    def use_optimized_model(self, flag=True):
        self._opt()["use_optimized_model"] = bool(flag)

    def enable_new_executor(self, x=True):
        self._opt()["new_executor"] = bool(x)

    def enable_new_ir(self, x=True):
        self._opt()["new_ir"] = bool(x)

    def new_ir_enabled(self):
        return self._opt().get("new_ir", True)

    def enable_profile(self):
        self._opt()["profile"] = True

    def enable_low_precision_io(self, x=True):
        self._opt()["low_precision_io"] = bool(x)

    def exp_enable_mixed_precision_ops(self, ops):
        self._opt().setdefault("mixed_white", set()).update(ops)

    def exp_disable_mixed_precision_ops(self, ops):
        self._opt().setdefault("mixed_black", set()).update(ops)

    def exp_enable_use_cutlass(self):
        self._opt()["cutlass"] = True

    def enable_cinn(self):
        self._opt()["cinn"] = True

    def memory_pool_init_size_mb(self):
        return self._opt().get("pool_mb", 100)

    def fraction_of_gpu_memory_for_pool(self):
        if not torch.cuda.is_available():
            return 0.0
        return self.memory_pool_init_size_mb() * (1 << 20) / torch.cuda.get_device_properties(self._gpu_id).total_memory

    def glog_info_disabled(self):
        return not self._glog

    def disable_mkldnn(self):
        self._opt()["mkldnn"] = False

    def mkldnn_enabled(self):
        return False

    def set_mkldnn_cache_capacity(self, n):
        pass

    def enable_mkldnn_bfloat16(self):
        self._precision = PrecisionType.Bfloat16

    def set_bfloat16_op(self, ops):
        self.exp_enable_mixed_precision_ops(ops)

    def set_model_buffer(self, prog_buffer, prog_size, params_buffer, params_size):
        """Model from memory: the two buffers are spooled to a private temp prefix and loaded from there."""
        import tempfile

        d = tempfile.mkdtemp(prefix="paddle_b200_infer_")
        with open(os.path.join(d, "m.pdmodel"), "wb") as f:
            f.write(bytes(prog_buffer)[:prog_size])
        with open(os.path.join(d, "m.pdiparams"), "wb") as f:
            f.write(bytes(params_buffer)[:params_size])
        self._prefix = os.path.join(d, "m")
        self._opt()["from_memory"] = True

    def model_from_memory(self):
        return self._opt().get("from_memory", False)

    def set_exec_stream(self, stream):
        self._opt()["exec_stream"] = stream

    def enable_tuned_tensorrt_dynamic_shape(self, path=None, allow_build_at_runtime=True):
        self._opt()["shape_range_info_path"] = path

    def tuned_tensorrt_dynamic_shape(self):
        return "shape_range_info_path" in self._opt()

    def collect_shape_range_info(self, path):
        self._opt()["collect_shape_range_info"] = path

    def shape_range_info_path(self):
        return self._opt().get("collect_shape_range_info", "")

    def shape_range_info_collected(self):
        return "collect_shape_range_info" in self._opt()

    def tensorrt_dynamic_shape_enabled(self):
        return False

    def tensorrt_precision_mode(self):
        return self._precision

    def enable_tensorrt_memory_optim(self, *a, **k):
        pass

    def enable_tensorrt_dla(self, *a, **k):
        pass

    def tensorrt_dla_enabled(self):
        return False

    def use_xpu(self):
        return False

    def enable_xpu(self, *a, **k):
        raise RuntimeError("XPU is not supported by paddle_b200 (sm_90a only)")

    def enable_custom_device(self, device_type, device_id=0, precision_mode=PrecisionType.Float32):
        raise RuntimeError(f"custom device '{device_type}' is not supported by paddle_b200 (sm_90a only)")

    def enable_onnxruntime(self):
        raise RuntimeError("onnxruntime is not part of this build; export with paddle.onnx.export and serve it externally")

    def onnxruntime_enabled(self):
        return False

    def disable_onnxruntime(self):
        pass

    def use_feed_fetch_ops_enabled(self):
        return False

    def specify_input_name(self):
        return True

    def to_native_config(self):
        return {"prefix": self._prefix, "use_gpu": self._use_gpu, "device": self._gpu_id, "precision": self._precision.name, **{k: v for k, v in self._opt().items()}}


class _Handle:
    """Input/output tensor handle (paddle_infer.Tensor)."""

    def __init__(self, name):
        self.name_, self._t = name, None

    def name(self):
        return self.name_

    def reshape(self, shape):
        self._shape = list(shape)

    def copy_from_cpu(self, arr):
        self._t = to_tensor(np.ascontiguousarray(arr))

    def share_external_data(self, t):
        self._t = t

    def copy_to_cpu(self):
        return self._t.numpy()

    def shape(self):
        return list(self._t.shape) if self._t is not None else getattr(self, "_shape", [])

    def type(self):
        return None if self._t is None else self._t.dtype

    def lod(self):
        return self._t.lod() if (self._t is not None and hasattr(self._t, "lod")) else getattr(self, "_lod", [])

    def set_lod(self, lod):
        self._lod = [list(l) for l in lod]
        if self._t is not None and hasattr(self._t, "set_lod"):
            self._t.set_lod(lod)

    def share_external_data_by_ptr_name(self, *a, **k):
        raise RuntimeError("raw pointer sharing is not exposed; use share_external_data(tensor)")

    def as_ndarray(self):
        return self.copy_to_cpu()

    def tolist(self):
        return self.copy_to_cpu().tolist()


class Predictor:
    def __init__(self, config):
        from .. import jit

        self._config = config
        self._layer = jit.load(config._prefix)
        spec = (getattr(self._layer, "_spec", None) or {}).get("input_spec") or []
        if not spec and hasattr(self._layer, "_blob"):   # traced-program artifact: feed names are recorded in the blob
            spec = [(None, None, n) for n in self._layer._blob["feeds"]]
        names = [s[2] if s and s[2] else f"x{i}" for i, s in enumerate(spec)] or ["x0"]
        self._inputs = {n: _Handle(n) for n in names}
        self._outputs = {}
        if config._use_gpu and torch.cuda.is_available():
            self._layer.to(torch.device("cuda", config._gpu_id))
            if config._precision in (PrecisionType.Half, PrecisionType.Bfloat16) and hasattr(self._layer, "_inner"):
                self._layer._inner._cast_floating(torch.float16 if config._precision == PrecisionType.Half else torch.bfloat16)
        self._dev = torch.device("cuda", config._gpu_id) if (config._use_gpu and torch.cuda.is_available()) else torch.device("cpu")
        self._ir_report = self._run_ir_passes()

    def _run_ir_passes(self):
        """Program artifacts go through the configured IR passes once, here (paddle_b200.pir); returns the per-pass report."""
        blob = getattr(self._layer, "_blob", None)
        passes = self._config._pir_passes()
        use_cinn = bool(self._config._opt().get("cinn"))           # Config.enable_cinn(): generated kernels for the elementwise / reduction chains
        if blob is None or not (passes or use_cinn):
            return []
        from .. import pir

        prog = blob["program"]
        if not pir.core_available() or any(n.kind != "op" for n in prog.nodes):
            return []
        try:
            opt, report = pir.optimize(prog, fetch_list=list(self._layer._fetch), passes=passes, return_report=True, cinn=False)
        except Exception:  # noqa: BLE001  (an op the translator cannot encode: run the program as saved)
            import os

            if os.environ.get("B200_JIT_DEBUG"):
                raise
            return []
        if self._config._opt().get("ir_debug"):
            for r in report:
                print(f"[ir pass] {r['pass']}: {r['ops_before']} -> {r['ops_after']} ops ({r['changed']} rewrites)")
        blob["program"] = opt
        if use_cinn:
            # generated kernels are compiled for concrete shapes and the saved program may declare dynamic ones: the Executor specialises it per
            # feed signature (first run generic, later runs compiled; static/__init__.py:Executor._specialised)
            opt.__dict__["_cinn_on_run"] = True
        return report

    def cinn_report(self):
        """{feed signature: FusionResult} of the specialisations built so far (Config.enable_cinn())."""
        prog = getattr(self._layer, "_blob", {}).get("program") if hasattr(self._layer, "_blob") else None
        out = {}
        for (_, sig, _n), p in (getattr(prog, "__dict__", {}).get("_cinn_cache", {}) or {}).items():
            rep = getattr(p, "__dict__", {}).get("_cinn_report")
            if rep is not None:
                out[sig] = rep
        return out

    def ir_pass_report(self):
        """[{pass, ops_before, ops_after, changed}] of the IR passes that ran when this predictor was built."""
        return list(self._ir_report)

    def get_input_names(self):
        return list(self._inputs)

    def get_input_handle(self, name):
        if name not in self._inputs:
            self._inputs[name] = _Handle(name)
        return self._inputs[name]

    def get_output_names(self):
        return list(self._outputs) or ["out0"]

    def get_output_handle(self, name):
        if name not in self._outputs:
            self._outputs[name] = _Handle(name)
        return self._outputs[name]

    @torch.no_grad()
    def run(self, inputs=None):
        if inputs is not None:
            args = [i if isinstance(i, torch.Tensor) else to_tensor(np.asarray(i)) for i in inputs]
        else:
            args = [h._t for h in self._inputs.values() if h._t is not None]
        p0 = next(iter(getattr(self._layer, "_inner", self._layer).parameters()), None)
        for hook in self.__dict__.get("_in_hooks", []):
            for n, a in zip(self._inputs, args):
                hook(n, a)
        args = [a.to(self._dev) for a in args]
        if p0 is not None and p0.dtype in (torch.float16, torch.bfloat16):
            args = [a.to(p0.dtype) if a.is_floating_point() else a for a in args]
        out = self._layer(*args)
        outs = list(out) if isinstance(out, (list, tuple)) else [out]
        for i, o in enumerate(outs):
            self.get_output_handle(f"out{i}")._t = o
            for hook in self.__dict__.get("_out_hooks", []):
                hook(f"out{i}", o)
        return outs if inputs is not None else True

    def clone(self, stream=None):
        return Predictor(self._config)

    def zero_copy_run(self):
        return self.run()

    def register_input_hook(self, hook):
        """hook(name, tensor) before every run. Parity: analysis_predictor RegisterInputHook."""
        self.__dict__.setdefault("_in_hooks", []).append(hook)

    def register_output_hook(self, hook):
        self.__dict__.setdefault("_out_hooks", []).append(hook)

    def get_serialized_program(self):
        with open(self._config._prefix + ".pdmodel", "rb") as f:
            return f.read()

    def clear_intermediate_tensor(self):
        pass

    def try_shrink_memory(self):
        if torch.cuda.is_available():
            torch.cuda.empty_cache()


def create_predictor(config):
    return Predictor(config)


class PredictorPool:
    def __init__(self, config, size=1):
        self._preds = [Predictor(config) for _ in range(size)]

    def retrive(self, idx):
        return self._preds[idx]

    retrieve = retrive


def get_version():
    from .. import __version__

    return f"paddle_b200 {__version__} (sm_90a)"


def get_trt_compile_version():
    return (0, 0, 0)


def get_trt_runtime_version():
    return (0, 0, 0)


def get_num_bytes_of_data_type(dtype):
    return {DataType.FLOAT32: 4, DataType.INT64: 8, DataType.INT32: 4, DataType.UINT8: 1, DataType.INT8: 1, DataType.FLOAT16: 2,
            DataType.BOOL: 1, DataType.FLOAT64: 8, DataType.BFLOAT16: 2}[dtype]


def convert_to_mixed_precision(model_file, params_file, mixed_model_file, mixed_params_file, mixed_precision, backend=None, keep_io_types=True, black_list=None, **kw):
    from .. import jit
    from ..framework.io import load, save

    prefix = model_file[: -len(".pdmodel")] if model_file.endswith(".pdmodel") else model_file
    sd = load(prefix + ".pdiparams")
    d = torch.float16 if mixed_precision == PrecisionType.Half else torch.bfloat16
    sd = {k: (v.astype(d) if isinstance(v, torch.Tensor) and v.is_floating_point() else v) for k, v in sd.items()}
    out = mixed_model_file[: -len(".pdmodel")] if mixed_model_file.endswith(".pdmodel") else mixed_model_file
    save(sd, out + ".pdiparams")
    import shutil

    shutil.copy(prefix + ".pdmodel", out + ".pdmodel")


Tensor = _Handle
XpuConfig = InternalUtils = None


def _get_phi_kernel_name(op_name):
    """Fluid op name -> phi kernel name (the two differ only for a handful of legacy ops)."""
    return {"matmul_v2": "matmul", "elementwise_add": "add", "elementwise_sub": "subtract", "elementwise_mul": "multiply", "elementwise_div": "divide",
            "reduce_sum": "sum", "reduce_mean": "mean", "fill_constant": "full", "lookup_table_v2": "embedding"}.get(op_name, op_name)
