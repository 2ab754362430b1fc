"""Weight-only quantised serving: `quantize_weights(model, algo, group_size, experts=False)` replaces the projection layers of a decoder-only
model of this package with `WeightOnlyLinear`, which holds int8 / int4 weights and fp32 scales and computes through
`nn.quant.weight_only_linear`; with experts=True a Mixtral model's stacked MoE experts become `WeightOnlyExpertFFN` in the same call.

The generation adapters (models/generation.py) call these layers as modules, so `generate()`, `LLMEngine` (chunked prefill, 8-bit KV
caches, prefix caching, a quantised draft model) and `calibrate_kv_cache` serve a quantised model unchanged.  On CUDA a step with at most
64 rows runs the in-SM dequantising GEMM (csrc/gemm_wo_sm100.cu); a larger step dequantises each weight once and runs the 16-bit GEMM.
Quantised experts follow the same split by routed slots (tokens x top-k): up to kernels.moe.WO_MOE_MAX_SLOTS they run the grouped in-SM
kernel over the selected experts only, above it each expert stack is dequantised in one launch for the 16-bit grouped GEMM.

`quantize_weights(model, "llm.int8", threshold=6.0)` replaces the same projections with `LLMInt8Linear` (int8 weights, int8 activations
quantised per token, `nn.quant.llm_int8_linear`): every step's GEMMs run on the int8 tensor cores, which is what pays off for prefill and
large batches.  threshold=float("inf") keeps all columns in int8 and is the sync-free path for serving (two launches per layer, no host
read); a finite threshold keeps outlier columns in 16-bit and reads their count on the host once per layer call.

Quantised layers:  Llama `qkv_proj, o_proj, gate_up_proj, down_proj`;  Mixtral `qkv_proj, o_proj`, and with experts=True its MoE experts
(the router stays 16-bit);  GPT `qkv, proj, fc1, fc2`.  Embeddings, norms and the LM head stay 16-bit.  Expert-parallel MoE layers cannot
hold quantised experts.  Inference only."""
from __future__ import annotations

import torch

from .. import nn
from ..incubate.moe import ExpertFFN, WeightOnlyExpertFFN
from ..nn import quant as Q
from ..tensor import Tensor

_ALGOS = {"weight_only_int8": "int8", "weight_only_int4": "int4"}
_ALL_ALGOS = sorted(_ALGOS) + ["llm.int8"]


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


class WeightOnlyLinear(nn.Layer):
    """y = x @ dequant(quant_weight)^T + bias.  `quant_weight` int8 [out, in] (int4: two per byte, [out, in / 2]) and `weight_scale` fp32
    [out] (per-channel) or [in / group_size, out] are buffers, not parameters: the layer has nothing to train, and a model's parameters
    still start with its 16-bit embedding.  The bias stays in the activation dtype."""

    def __init__(self, linear, algo="weight_only_int8", group_size=-1):
        super().__init__()
        w = _raw(linear.weight).detach()                         # [in, out]
        self.in_features, self.out_features = int(w.shape[0]), int(w.shape[1])
        self.algo, self.weight_dtype, self.group_size = algo, _ALGOS[algo], int(group_size)
        q, s = Q.weight_quantize(w.float().as_subclass(Tensor), algo=algo, group_size=self.group_size)
        self.register_buffer("quant_weight", _raw(q))
        self.register_buffer("weight_scale", _raw(s).float().contiguous())
        self.register_buffer("bias", None if linear.bias is None else _raw(linear.bias).detach().clone())

    def forward(self, x):
        return Q.weight_only_linear(x, self.quant_weight, self.bias, self.weight_scale, self.weight_dtype, group_size=self.group_size)

    def dequantized_weight(self, dtype=None):
        """The [in, out] weight this layer computes with, in `dtype` (default: the bias's dtype, else fp32)."""
        if dtype is None:
            dtype = self.bias.dtype if self.bias is not None else torch.float32
        return Q.weight_dequantize(self.quant_weight, self.weight_scale, self.algo, dtype, self.group_size)

    def extra_repr(self):
        g = "per-channel" if self.group_size <= 0 else f"group_size={self.group_size}"
        return f"in_features={self.in_features}, out_features={self.out_features}, {self.weight_dtype}, {g}"


class LLMInt8Linear(nn.Layer):
    """y = llm_int8_linear(x, quant_weight, bias, weight_scale, threshold).  `quant_weight` int8 [out, in] and `weight_scale` fp32 [out]
    (from `weight_quantize(algo="llm.int8")`) and the bias (activation dtype) are buffers."""

    def __init__(self, linear, threshold=6.0):
        super().__init__()
        w = _raw(linear.weight).detach()                         # [in, out]
        self.in_features, self.out_features = int(w.shape[0]), int(w.shape[1])
        self.threshold = float(threshold)
        q, s = Q.weight_quantize(w.float().as_subclass(Tensor), algo="llm.int8")
        self.register_buffer("quant_weight", _raw(q))
        self.register_buffer("weight_scale", _raw(s).float().contiguous())
        self.register_buffer("bias", None if linear.bias is None else _raw(linear.bias).detach().clone())

    def forward(self, x):
        return Q.llm_int8_linear(x, self.quant_weight, self.bias, self.weight_scale, self.threshold)

    def dequantized_weight(self, dtype=None):
        """The [in, out] weight of the int8 GEMM, in `dtype` (default: the bias's dtype, else fp32)."""
        if dtype is None:
            dtype = self.bias.dtype if self.bias is not None else torch.float32
        return Q.weight_dequantize(self.quant_weight, self.weight_scale, "weight_only_int8", dtype)

    def extra_repr(self):
        return f"in_features={self.in_features}, out_features={self.out_features}, llm.int8, threshold={self.threshold}"


def _targets(model):
    """(parent layer, attribute name) of every projection `quantize_weights` replaces."""
    if hasattr(model, "gpt") and hasattr(model.gpt, "blocks"):
        return [(blk, n) for blk in model.gpt.blocks for n in ("qkv", "proj", "fc1", "fc2")]
    if hasattr(model, "llama"):
        return [(p, n) for layer in model.llama.layers
                for p, names in ((layer.self_attn, ("qkv_proj", "o_proj")), (layer.mlp, ("gate_up_proj", "down_proj"))) for n in names]
    if hasattr(model, "embed_tokens") and hasattr(model, "layers") and hasattr(list(model.layers)[0], "moe"):
        return [(layer.self_attn, n) for layer in model.layers for n in ("qkv_proj", "o_proj")]
    raise ValueError(f"quantize_weights does not know the layout of {type(model).__name__}")


def _moe_layers(model):
    """The MoELayer of every decoder layer (Mixtral), or [] for a dense model."""
    if hasattr(model, "embed_tokens") and hasattr(model, "layers") and hasattr(list(model.layers)[0], "moe"):
        return [layer.moe for layer in model.layers]
    return []


def quantize_weights(model, algo="weight_only_int8", group_size=-1, experts=False, threshold=6.0):
    """Replace the model's projection layers in place with `WeightOnlyLinear` (int8 or int4 weights, per-channel scales for group_size -1,
    else one scale per `group_size` consecutive inputs of a channel) and return the model.  experts=True also replaces the stacked MoE
    experts of a Mixtral model (`ExpertFFN`) with `WeightOnlyExpertFFN`.  algo="llm.int8" installs `LLMInt8Linear` instead (int8 weights
    and per-token int8 activations, outlier columns above `threshold` in 16-bit; threshold=float("inf") is the sync-free serving path);
    it takes per-channel scales only, needs in_features % 16 == 0 and does not quantize experts.  Every check runs before any layer
    changes."""
    if algo not in _ALL_ALGOS:
        raise ValueError(f"algo must be one of {_ALL_ALGOS}, got {algo!r}")
    llm_int8 = algo == "llm.int8"
    if group_size not in (-1, 64, 128):
        raise ValueError(f"group_size must be -1 (per-channel), 64 or 128, got {group_size!r}")
    if llm_int8 and group_size != -1:
        raise ValueError("llm.int8 uses per-channel weight scales: group_size must be -1")
    if llm_int8 and experts:
        raise ValueError("llm.int8 does not quantize MoE experts (experts=True)")
    targets = _targets(model)
    moes = _moe_layers(model) if experts else []
    if experts and not moes:
        raise ValueError(f"experts=True: {type(model).__name__} has no MoE experts")
    for moe in moes:
        if moe.world_size > 1:
            raise ValueError("experts=True: expert-parallel MoE layers (world_size > 1) cannot hold quantized experts")
        if isinstance(moe.experts, WeightOnlyExpertFFN):
            raise ValueError("the model is already quantized")
        if not isinstance(moe.experts, ExpertFFN):
            raise ValueError(f"experts=True replaces stacked ExpertFFN experts; found {type(moe.experts).__name__}")
        ex = moe.experts
        for name, k in (("ffn1", int(ex.w1.shape[1])), ("ffn2", int(ex.w2.shape[1]))):
            if group_size > 0 and k % group_size:
                raise ValueError(f"experts {name}: fan-in {k} is not a multiple of group_size {group_size}")
            if algo == "weight_only_int4" and k % 2:
                raise ValueError(f"experts {name}: int4 packs two inputs per byte, fan-in {k} is odd")
    for parent, name in targets:
        layer = getattr(parent, name)
        if isinstance(layer, (WeightOnlyLinear, LLMInt8Linear)):
            raise ValueError("the model is already quantized")
        if not isinstance(layer, nn.Linear):
            raise ValueError(f"quantize_weights replaces nn.Linear layers; {name} is a {type(layer).__name__}")
        k = layer.in_features
        if group_size > 0 and k % group_size:
            raise ValueError(f"{name}: in_features {k} is not a multiple of group_size {group_size}")
        if algo == "weight_only_int4" and k % 2:
            raise ValueError(f"{name}: int4 packs two inputs per byte, in_features {k} is odd")
        if llm_int8 and k % 16:
            raise ValueError(f"{name}: llm.int8 needs in_features % 16 == 0, got {k}")
    with torch.no_grad():
        for parent, name in targets:
            lin = getattr(parent, name)
            setattr(parent, name, LLMInt8Linear(lin, threshold) if llm_int8 else WeightOnlyLinear(lin, algo, group_size))
        for moe in moes:
            moe.experts = WeightOnlyExpertFFN(moe.experts, algo, group_size)
    return model
