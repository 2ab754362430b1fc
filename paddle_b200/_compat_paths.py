"""Import-path compatibility: every dotted module path a user of the reference imports from resolves here.

Two mechanisms, both through one meta-path finder:
  * after `install_as_paddle()`, `import paddle.x.y` is served by importing `paddle_b200.x.y` and aliasing it (one module object,
    never a second copy with duplicated global state);
  * reference paths whose code lives elsewhere in this tree (`paddle.distributed.fleet.meta_parallel`, `paddle.tensor.math`,
    `paddle.incubate.distributed.models.moe`, `paddle.nn.functional.flash_attention`, ...) are synthesised as small modules that
    re-export the real objects."""
from __future__ import annotations

import importlib
import importlib.abc
import importlib.machinery
import sys
import types

_PKG = __name__.rsplit(".", 1)[0]          # "paddle_b200"
_ALIASES = {}                                # relative dotted path -> factory() -> module


def alias(path):
    def deco(fn):
        _ALIASES[path] = fn
        return fn
    return deco


def _mod(name, doc, **attrs):
    m = types.ModuleType(name, doc)
    m.__dict__.update(attrs)
    m.__path__ = []           # lets `import a.b.c` continue below a synthesised module
    return m


def _reexport(path, doc, sources, names=None, extra=None):
    """Module `path` exposing `names` (or every public name) looked up in `sources` (dotted module paths relative to the package)."""
    def factory():
        mods = [importlib.import_module(_PKG + "." + s if s else _PKG) for s in sources]
        m = _mod(_PKG + "." + path, doc)
        if names is None:
            for src in reversed(mods):
                for k in getattr(src, "__all__", None) or [k for k in vars(src) if not k.startswith("_")]:
                    if hasattr(src, k):
                        setattr(m, k, getattr(src, k))
        else:
            for k in names:
                for src in mods:
                    if hasattr(src, k):
                        setattr(m, k, getattr(src, k))
                        break
        for k, v in (extra() if extra else {}).items():
            setattr(m, k, v)
        return m
    _ALIASES[path] = factory


# ---- paddle.tensor.* (the reference splits the op namespace into files) ---------------------------------------------------------
for _sub, _src in (("math", "ops.math"), ("manipulation", "ops.manipulation"), ("creation", "ops.creation"), ("linalg", "ops.linalg"), ("logic", "ops.logic"),
                   ("search", "ops.search"), ("stat", "ops.stat"), ("random", "ops.random"), ("einsum", "ops.einsum"), ("attribute", "ops"), ("ops", "ops"),
                   ("to_string", "ops")):
    _reexport("tensor." + _sub, f"paddle.tensor.{_sub}", [_src])

# ---- autograd / hapi / jit / nn / text / static sub-paths -------------------------------------------------------------------------
_reexport("autograd.py_layer", "paddle.autograd.py_layer", ["autograd"], ["PyLayer", "PyLayerContext", "once_differentiable"])
_reexport("autograd.backward_mode", "paddle.autograd.backward_mode", ["autograd"], ["backward"])
_reexport("autograd.autograd", "paddle.autograd.autograd", ["autograd"], ["jacobian", "hessian"])
_reexport("hapi.callbacks", "paddle.hapi.callbacks", ["callbacks"])
_reexport("hapi.model_summary", "paddle.hapi.model_summary", ["hapi.summary"])
_reexport("hapi.dynamic_flops", "paddle.hapi.dynamic_flops", ["hapi"], ["flops"])
_reexport("jit.dy2static", "paddle.jit.dy2static (capture here is CUDA-graph based; see jit/__init__.py)", ["jit"])
_reexport("jit.api", "paddle.jit.api", ["jit"])
_reexport("jit.translated_layer", "paddle.jit.translated_layer", ["jit"], ["TranslatedLayer"])
_reexport("nn.functional.flash_attention", "paddle.nn.functional.flash_attention", ["nn.functional.attention", "nn.functional"],
          ["flash_attention", "flash_attn_unpadded", "flash_attn_qkvpacked", "flash_attn_varlen_qkvpacked", "flashmask_attention", "scaled_dot_product_attention",
           "sdp_kernel", "calc_reduced_attention_scores", "flash_attention_with_sparse_mask"])
_reexport("nn.functional.pooling", "paddle.nn.functional.pooling", ["nn.functional.conv_pool_norm"])
_reexport("nn.functional.conv", "paddle.nn.functional.conv", ["nn.functional.conv_pool_norm"])
_reexport("nn.functional.norm", "paddle.nn.functional.norm", ["nn.functional.conv_pool_norm"])
_reexport("nn.functional.input", "paddle.nn.functional.input", ["nn.functional"], ["one_hot", "embedding"])
_reexport("nn.functional.vision", "paddle.nn.functional.vision", ["nn.functional"], ["affine_grid", "grid_sample", "pixel_shuffle", "pixel_unshuffle", "channel_shuffle"])
_reexport("nn.functional.distance", "paddle.nn.functional.distance", ["nn.functional"], ["pairwise_distance", "pdist"])
_reexport("nn.functional.extension", "paddle.nn.functional.extension", ["nn.functional"], ["diag_embed", "sequence_mask", "gather_tree", "temporal_shift"])
_reexport("nn.layer.common", "paddle.nn.layer.common", ["nn.common", "nn"])
_reexport("nn.layer.layers", "paddle.nn.layer.layers", ["nn.layer"], ["Layer"])
_reexport("nn.layer.activation", "paddle.nn.layer.activation", ["nn.activation_loss"])
_reexport("nn.layer.loss", "paddle.nn.layer.loss", ["nn.activation_loss"])
_reexport("nn.layer.conv", "paddle.nn.layer.conv", ["nn.conv_norm_pool"])
_reexport("nn.layer.norm", "paddle.nn.layer.norm", ["nn.conv_norm_pool"])
_reexport("nn.layer.pooling", "paddle.nn.layer.pooling", ["nn.conv_norm_pool"])
_reexport("nn.layer.rnn", "paddle.nn.layer.rnn", ["nn.rnn"])
_reexport("nn.layer.transformer", "paddle.nn.layer.transformer", ["nn.transformer"])
_reexport("nn.layer.container", "paddle.nn.layer.container", ["nn"], ["Sequential", "LayerList", "LayerDict", "ParameterList", "ParameterDict"])
_reexport("text.datasets", "paddle.text.datasets", ["text"], ["Conll05st", "Imdb", "Imikolov", "Movielens", "UCIHousing", "WMT14", "WMT16"])
_reexport("text.viterbi_decode", "paddle.text.viterbi_decode", ["text"], ["ViterbiDecoder", "viterbi_decode"])
_reexport("static.quantization", "paddle.static.quantization", ["quantization"])
_reexport("static.io", "paddle.static.io", ["static"], ["save", "load", "save_inference_model", "load_inference_model", "serialize_program", "deserialize_program",
                                                      "serialize_persistables", "deserialize_persistables", "save_to_file", "load_from_file", "normalize_program",
                                                      "load_program_state", "set_program_state"])
_reexport("optimizer.optimizer", "paddle.optimizer.optimizer", ["optimizer"], ["Optimizer"])
_reexport("optimizer.adamw", "paddle.optimizer.adamw", ["optimizer"], ["AdamW"])
_reexport("optimizer.adam", "paddle.optimizer.adam", ["optimizer"], ["Adam"])
_reexport("optimizer.momentum", "paddle.optimizer.momentum", ["optimizer"], ["Momentum"])
_reexport("optimizer.sgd", "paddle.optimizer.sgd", ["optimizer"], ["SGD"])
_reexport("io.dataloader.dataset", "paddle.io.dataloader.dataset", ["io.dataset"])
_reexport("io.dataloader.sampler", "paddle.io.dataloader.sampler", ["io.sampler"])
_reexport("io.dataloader.batch_sampler", "paddle.io.dataloader.batch_sampler", ["io.sampler"], ["BatchSampler", "DistributedBatchSampler"])
_reexport("io.dataloader.collate", "paddle.io.dataloader.collate", ["io"], ["default_collate_fn", "default_convert_fn"])
_reexport("io.dataloader.worker", "paddle.io.dataloader.worker", ["io"], ["get_worker_info"])
_reexport("vision.transforms.functional", "paddle.vision.transforms.functional", ["vision.transforms"])
_reexport("vision.transforms.transforms", "paddle.vision.transforms.transforms", ["vision.transforms"])
_reexport("base.param_attr", "paddle.base.param_attr", ["nn.layer", "static"], ["ParamAttr", "WeightNormParamAttr"])
_reexport("base.executor", "paddle.base.executor", ["static"], ["Executor", "global_scope", "scope_guard"])
_reexport("base.data_feeder", "paddle.base.data_feeder", ["framework.dtype"], ["convert_dtype"])
_reexport("base.layer_helper", "paddle.base.layer_helper", ["nn.layer"], ["_make_parameter"])
_reexport("framework.random", "paddle.framework.random", ["framework.random", ""], ["seed", "get_rng_state", "set_rng_state", "get_cuda_rng_state", "set_cuda_rng_state"])


# ---- distributed paths ------------------------------------------------------------------------------------------------------------
_FLEET = "distributed.fleet"
_reexport(_FLEET + ".meta_parallel", "paddle.distributed.fleet.meta_parallel", [_FLEET + ".mp_layers", _FLEET + ".pipeline", _FLEET + ".hybrid", _FLEET + ".random"])
_reexport(_FLEET + ".meta_parallel.parallel_layers", "fleet.meta_parallel.parallel_layers", [_FLEET + ".mp_layers", _FLEET + ".pipeline", _FLEET + ".random"])
_reexport(_FLEET + ".meta_parallel.parallel_layers.pp_layers", "pp_layers", [_FLEET + ".pipeline"], ["PipelineLayer", "LayerDesc", "SharedLayerDesc", "SegmentLayers"])
_reexport(_FLEET + ".meta_parallel.parallel_layers.mp_layers", "mp_layers", [_FLEET + ".mp_layers"])
_reexport(_FLEET + ".meta_parallel.parallel_layers.random", "random", [_FLEET + ".random"])
_reexport(_FLEET + ".meta_parallel.pipeline_parallel", "pipeline_parallel", [_FLEET + ".pipeline"], ["PipelineParallel", "PipelineParallelWithInterleave", "PipelineParallelWithInterleaveFthenB", "PipelineParallelZeroBubble"])
_reexport(_FLEET + ".meta_parallel.tensor_parallel", "tensor_parallel", [_FLEET + ".hybrid"], ["TensorParallel"])
_reexport(_FLEET + ".meta_parallel.sharding_parallel", "sharding_parallel", [_FLEET + ".hybrid"], ["ShardingParallel"])
_reexport(_FLEET + ".meta_parallel.segment_parallel", "segment_parallel", [_FLEET + ".hybrid"], ["SegmentParallel"])
_reexport(_FLEET + ".meta_parallel.pp_utils", "pp_utils", [_FLEET + ".pipeline"])
_reexport(_FLEET + ".meta_parallel.pp_utils.p2p_communication", "p2p_communication", [_FLEET + ".pipeline"])
_reexport(_FLEET + ".meta_parallel.sharding", "fleet.meta_parallel.sharding", ["distributed.sharding"])
_reexport(_FLEET + ".meta_parallel.sharding.group_sharded_stage2", "group_sharded_stage2", ["distributed.sharding"], ["GroupShardedStage2"])
_reexport(_FLEET + ".meta_parallel.sharding.group_sharded_stage3", "group_sharded_stage3", ["distributed.sharding"], ["GroupShardedStage3"])
_reexport(_FLEET + ".meta_parallel.sharding.group_sharded_optimizer_stage2", "group_sharded_optimizer_stage2", ["distributed.sharding"], ["GroupShardedOptimizerStage2"])
_reexport(_FLEET + ".meta_parallel.sharding.group_sharded_utils", "group_sharded_utils", ["distributed.sharding"], ["GroupShardedScaler", "GroupShardedClipGrad"])
_reexport(_FLEET + ".layers", "paddle.distributed.fleet.layers", [_FLEET + ".mp_layers"])
_reexport(_FLEET + ".layers.mpu", "paddle.distributed.fleet.layers.mpu", [_FLEET + ".mp_layers", _FLEET + ".random"])
_reexport(_FLEET + ".layers.mpu.mp_layers", "mpu.mp_layers", [_FLEET + ".mp_layers"])
_reexport(_FLEET + ".layers.mpu.mp_ops", "mpu.mp_ops", [_FLEET + ".mp_layers", "distributed"],
          ["_c_identity", "_mp_allreduce", "_c_concat", "_c_split", "split", "ParallelCrossEntropy", "ScatterOp", "GatherOp", "AllGatherOp", "ReduceScatterOp"])
_reexport(_FLEET + ".layers.mpu.random", "mpu.random", [_FLEET + ".random"])
_reexport(_FLEET + ".base", "paddle.distributed.fleet.base", [_FLEET + ".topology", _FLEET + ".strategy", _FLEET + ".base_extras"])
_reexport(_FLEET + ".base.topology", "fleet.base.topology", [_FLEET + ".topology"])
_reexport(_FLEET + ".base.distributed_strategy", "fleet.base.distributed_strategy", [_FLEET + ".strategy"])
_reexport(_FLEET + ".base.role_maker", "fleet.base.role_maker", [_FLEET + ".base_extras", _FLEET], ["Role", "PaddleCloudRoleMaker", "UserDefinedRoleMaker"])
_reexport(_FLEET + ".base.util_factory", "fleet.base.util_factory", [_FLEET + ".base_extras"], ["UtilBase"])
_reexport(_FLEET + ".meta_optimizers", "fleet.meta_optimizers", [_FLEET + ".hybrid", "distributed.sharding"],
          ["HybridParallelOptimizer", "HybridParallelClipGrad", "DygraphShardingOptimizer", "HybridParallelGradScaler"])
_reexport(_FLEET + ".meta_optimizers.dygraph_optimizer", "dygraph_optimizer", [_FLEET + ".hybrid", "distributed.sharding"],
          ["HybridParallelOptimizer", "HybridParallelClipGrad", "DygraphShardingOptimizer", "HybridParallelGradScaler"])
_reexport(_FLEET + ".meta_optimizers.dygraph_optimizer.hybrid_parallel_optimizer", "hybrid_parallel_optimizer", [_FLEET + ".hybrid"],
          ["HybridParallelOptimizer", "HybridParallelClipGrad"])
_reexport(_FLEET + ".data_generator", "fleet.data_generator", [_FLEET + ".base_extras"], ["MultiSlotDataGenerator", "MultiSlotStringDataGenerator"])
_reexport(_FLEET + ".dataset", "fleet.dataset", ["distributed.extras"], ["InMemoryDataset", "QueueDataset"])
_reexport(_FLEET + ".scaler", "fleet.scaler", [_FLEET], ["distributed_scaler"])
_reexport(_FLEET + ".auto", "paddle.distributed.fleet.auto (semi-auto parallel entry points)", ["distributed.auto_parallel"])
_reexport(_FLEET + ".fleet", "fleet.fleet", [_FLEET + ".base_extras", _FLEET], ["Fleet"])
_reexport("distributed.parallel", "paddle.distributed.parallel", ["distributed", "distributed.data_parallel"], ["DataParallel", "init_parallel_env", "ParallelEnv", "get_rank", "get_world_size"])
_reexport("distributed.collective", "paddle.distributed.collective", ["distributed.collective"])
_reexport("distributed.communication.stream", "paddle.distributed.communication.stream", ["distributed.stream"])
_reexport("distributed.auto_parallel.static", "auto_parallel.static", ["distributed.auto_parallel"])
_reexport("distributed.checkpoint.save_state_dict", "checkpoint.save_state_dict", ["distributed.checkpoint"], ["save_state_dict"])
_reexport("distributed.checkpoint.load_state_dict", "checkpoint.load_state_dict", ["distributed.checkpoint"], ["load_state_dict"])
_reexport("distributed.utils", "paddle.distributed.utils", ["distributed.dist_utils", "incubate.moe"])
_reexport("distributed.utils.moe_utils", "distributed.utils.moe_utils", ["incubate.moe"], ["global_scatter", "global_gather"])
_reexport("distributed.models", "paddle.distributed.models", [])
_reexport("distributed.models.moe", "paddle.distributed.models.moe", ["incubate.moe"])

@alias("incubate.asp")
def _asp_module():
    inc = importlib.import_module(_PKG + ".incubate")
    a = inc.__dict__["asp"]
    m = _mod(_PKG + ".incubate.asp", "paddle.incubate.asp: 2:4 structured sparsity")
    for k in ("calculate_density", "decorate", "prune_model", "set_excluded_layers", "reset_excluded_layers", "add_supported_layer"):
        if hasattr(a, k):
            setattr(m, k, getattr(a, k))
    return m


_reexport("geometric.message_passing", "paddle.geometric.message_passing", ["geometric"], ["send_u_recv", "send_ue_recv", "send_uv"])
_reexport("geometric.sampling", "paddle.geometric.sampling", ["geometric"], ["sample_neighbors", "weighted_sample_neighbors"])
_reexport("geometric.reindex", "paddle.geometric.reindex", ["geometric"], ["reindex_graph", "reindex_heter_graph"])
_reexport("geometric.math", "paddle.geometric.math", ["geometric"], ["segment_sum", "segment_mean", "segment_min", "segment_max"])
_reexport("base.layers", "paddle.base.layers (legacy op-builder namespace)", ["static.nn", "ops"])
_reexport(_FLEET + ".runtime", "paddle.distributed.fleet.runtime", [_FLEET + ".ps_mode"])


@alias("device.xpu")
def _xpu_module():
    def _none(*a, **k):
        raise RuntimeError("XPU devices are not supported by paddle_b200 (sm_90a only)")

    return _mod(_PKG + ".device.xpu", "paddle.device.xpu: not available on this target", synchronize=_none, device_count=lambda: 0, set_debug_level=lambda level=1: None,
                empty_cache=lambda: None, max_memory_allocated=lambda device=None: 0, memory_allocated=lambda device=None: 0)


# ---- incubate paths ---------------------------------------------------------------------------------------------------------------
_reexport("incubate.distributed", "paddle.incubate.distributed", [])
_reexport("incubate.distributed.fleet", "paddle.incubate.distributed.fleet", [_FLEET + ".recompute"], ["recompute_sequential", "recompute_hybrid"])
_reexport("incubate.distributed.models", "paddle.incubate.distributed.models", [])
_reexport("incubate.distributed.models.moe", "paddle.incubate.distributed.models.moe", ["incubate.moe"])
_reexport("incubate.distributed.models.moe.moe_layer", "moe_layer", ["incubate.moe"], ["MoELayer"])
_reexport("incubate.distributed.models.moe.gate", "moe.gate", ["incubate.moe"], ["BaseGate", "NaiveGate", "GShardGate", "SwitchGate"])
_reexport("incubate.distributed.models.moe.grad_clip", "moe.grad_clip", ["incubate.moe"], ["ClipGradForMOEByGlobalNorm"])
_reexport("incubate.distributed.utils", "paddle.incubate.distributed.utils", [])
_reexport("incubate.distributed.utils.io", "incubate.distributed.utils.io", ["distributed.extras"], ["save_for_auto_inference"])
_reexport("incubate.optimizer.functional", "paddle.incubate.optimizer.functional", ["incubate.optimizer_functional"], ["minimize_bfgs", "minimize_lbfgs"])
_reexport("incubate.tensor", "paddle.incubate.tensor", ["geometric"], ["segment_sum", "segment_mean", "segment_max", "segment_min"])
_reexport("incubate.tensor.math", "paddle.incubate.tensor.math", ["geometric"], ["segment_sum", "segment_mean", "segment_max", "segment_min"])
_reexport("incubate.operators", "paddle.incubate.operators", ["incubate"],
          ["softmax_mask_fuse", "softmax_mask_fuse_upper_triangle", "graph_send_recv", "graph_khop_sampler", "graph_sample_neighbors", "graph_reindex"])
_reexport("incubate.framework", "paddle.incubate.framework", ["framework.random", ""], ["get_rng_state", "set_rng_state", "seed"])
_reexport("incubate.passes", "paddle.incubate.passes", [], extra=lambda: {"ir": _reexport_now("static.passes", ["register_pass", "PassManager", "new_pass"], RegisterPass="register_pass")})
_reexport("incubate.nn.functional.fused_transformer", "fused_transformer", ["incubate.nn.functional"])
_reexport("incubate.nn.layer", "paddle.incubate.nn.layer", ["incubate.nn"])
_reexport("incubate.nn.layer.fused_transformer", "incubate.nn.layer.fused_transformer", ["incubate.nn"])


def _reexport_now(src, names, **renames):
    s = importlib.import_module(_PKG + "." + src)
    m = _mod(_PKG + ".incubate.passes.ir", "paddle.incubate.passes.ir")
    for k in names:
        setattr(m, k, getattr(s, k))
    for new, old in renames.items():
        setattr(m, new, getattr(s, old))
    return m


class _CallableModule(types.ModuleType):
    """A synthesised sub-module whose name is also a function of its parent (`paddle.text.viterbi_decode`, `F.flash_attention`):
    importing the module rebinds the parent attribute to it, so it keeps behaving as that function when called."""

    def __call__(self, *args, **kwargs):
        return self.__dict__["_shadowed"](*args, **kwargs)


class _Finder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    def find_spec(self, fullname, path=None, target=None):
        if fullname.startswith(_PKG + "."):
            rel = fullname[len(_PKG) + 1:]
            if rel in _ALIASES and not self._real_exists(fullname):
                return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        elif fullname.startswith("paddle.") and sys.modules.get("paddle") is sys.modules.get(_PKG):
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    @staticmethod
    def _real_exists(fullname):
        try:
            return importlib.machinery.PathFinder.find_spec(fullname.rsplit(".", 1)[1], getattr(sys.modules.get(fullname.rsplit(".", 1)[0]), "__path__", None) or []) is not None
        except Exception:
            return False

    def create_module(self, spec):
        name = spec.name
        if name.startswith("paddle."):
            return importlib.import_module(_PKG + name[len("paddle"):])      # the one and only module object, under a second name
        m = _ALIASES[name[len(_PKG) + 1:]]()
        parent = sys.modules.get(name.rsplit(".", 1)[0])
        shadowed = vars(parent).get(name.rsplit(".", 1)[1]) if parent is not None else None      # vars(): no lazy __getattr__ re-entry
        if shadowed is not None and callable(shadowed) and not isinstance(shadowed, types.ModuleType):
            cm = _CallableModule(m.__name__, m.__doc__)
            cm.__dict__.update({k: v for k, v in m.__dict__.items() if k not in ("__name__", "__doc__")})
            cm.__dict__["_shadowed"] = shadowed
            if getattr(shadowed, "__name__", None) and shadowed.__name__ not in cm.__dict__:
                cm.__dict__[shadowed.__name__] = shadowed
            m = cm
        return m

    def exec_module(self, module):
        pass


_finder = _Finder()


def install():
    if _finder not in sys.meta_path:
        sys.meta_path.insert(0, _finder)
    # plain modules that the reference has as packages: give them an (empty) search path so `import pkg.mod.sub` reaches the finder
    import os

    root = os.path.dirname(os.path.abspath(__file__))
    for rel in {p.rsplit(".", 1)[0] for p in _ALIASES if "." in p}:
        m = sys.modules.get(_PKG + "." + rel)
        if m is None and os.path.isfile(os.path.join(root, *rel.split(".")) + ".py"):
            m = importlib.import_module(_PKG + "." + rel)      # single-file module in this tree, package in the reference
        if m is not None and not hasattr(m, "__path__"):
            m.__path__ = []
