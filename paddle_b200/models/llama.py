"""Llama-2 family on paddle_b200 (fleet tensor/sequence/pipeline parallel aware).

Parity (role): the Llama used by the reference's hybrid-parallel benchmarks (test/auto_parallel/hybrid_strategy/
semi_auto_llama.py; PaddleNLP llama modeling on fleet mpu layers + incubate fused ops).  Every hot op is one of this
repo's sm_90a kernels: fused QKV / gate-up GEMMs (wgmma), in-place packed rotary, fused residual-add+RMSNorm,
SwiGLU, fused softmax-CE; row-parallel GEMMs go through parallel.fused_mp (GEMM + collective over peer memory).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from .. import nn
from ..distributed.fleet import mp_layers as mpu
from ..distributed.fleet import topology as topo
from ..distributed.fleet.recompute import recompute
from ..kernels import activation as KA
from ..kernels import attention as KAT
from ..kernels import loss as KL
from ..kernels import norm as KN
from ..kernels import rope as KR
from ..nn import functional as F
from ..nn import initializer as I
from ..tensor import Tensor


@dataclass
class LlamaConfig:
    vocab_size: int = 32000
    hidden_size: int = 5120
    intermediate_size: int = 13824
    num_hidden_layers: int = 40
    num_attention_heads: int = 40
    num_key_value_heads: int = 40
    max_position_embeddings: int = 4096
    rms_norm_eps: float = 1e-5
    rope_theta: float = 10000.0
    initializer_range: float = 0.02
    tensor_parallel_degree: int = 1
    sequence_parallel: bool = False
    recompute: bool = False
    recompute_skip_layers: int = 0      # the last k layers of a stage keep their activations (memory permitting)
    tie_word_embeddings: bool = False
    lean_activations: bool = True       # single-GPU: fused norm->linear / swiglu->linear nodes that do not keep the intermediate
    dtype: str = "bfloat16"

    @property
    def head_dim(self):
        return self.hidden_size // self.num_attention_heads


def llama2_13b(**kw):
    return LlamaConfig(**kw)


def llama2_7b(**kw):
    return LlamaConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32, num_attention_heads=32, num_key_value_heads=32, **kw)


def llama_tiny(**kw):
    base = dict(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=4,
                max_position_embeddings=128)
    base.update(kw)
    return LlamaConfig(**base)


def _mp_degree():
    hcg = topo.get_hybrid_communicate_group()
    return hcg.get_model_parallel_world_size() if hcg is not None else 1


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


def _w(t):
    return t.as_subclass(Tensor) if isinstance(t, torch.Tensor) and not isinstance(t, Tensor) else t


class LlamaRMSNorm(nn.Layer):
    def __init__(self, config):
        super().__init__()
        self.eps = config.rms_norm_eps
        self.weight = self.create_parameter([config.hidden_size], default_initializer=I.Constant(1.0))
        if config.sequence_parallel:
            mpu.mark_as_sequence_parallel_parameter(self.weight)

    def forward(self, x, residual=None):
        return KN.rms_norm(x, self.weight, self.eps, residual=residual)


class LlamaAttention(nn.Layer):
    def __init__(self, config):
        super().__init__()
        self.config = config
        mp = _mp_degree()
        self.mp = mp
        self.num_heads = config.num_attention_heads // mp
        self.num_kv_heads = config.num_key_value_heads // mp
        self.head_dim = config.head_dim
        h = config.hidden_size
        kv = config.num_key_value_heads * self.head_dim
        std = config.initializer_range
        wattr = nn.ParamAttr(initializer=I.Normal(0.0, std))
        oattr = nn.ParamAttr(initializer=I.Normal(0.0, std / math.sqrt(2 * config.num_hidden_layers)))
        # fused QKV projection: per mp-rank columns are laid out (q heads | k heads | v heads)
        if mp > 1:
            Col = mpu.ColumnSequenceParallelLinear if config.sequence_parallel else mpu.ColumnParallelLinear
            Row = mpu.RowSequenceParallelLinear if config.sequence_parallel else mpu.RowParallelLinear
            self.qkv_proj = Col(h, h + 2 * kv, weight_attr=wattr, has_bias=False, gather_output=False)
            self.o_proj = Row(h, h, weight_attr=oattr, has_bias=False, input_is_parallel=True)
        else:
            self.qkv_proj = nn.Linear(h, h + 2 * kv, weight_attr=wattr, bias_attr=False)
            self.o_proj = nn.Linear(h, h, weight_attr=oattr, bias_attr=False)

    def forward(self, x, cos, sin, position_ids=None):
        return self.attend(self.qkv_proj(x), cos, sin, position_ids)

    def attend(self, qkv, cos, sin, position_ids=None):
        """Everything after the QKV projection: rotary, attention, output projection."""
        cfg = self.config
        nh, nkv, hd = self.num_heads, self.num_kv_heads, self.head_dim
        total = nh + 2 * nkv
        if cfg.sequence_parallel and self.mp > 1 and position_ids is None and _raw(qkv).is_cuda:
            # sequence-parallel layout [S, B, *] is kept end to end: rotary gets explicit positions (token t = s*B + b -> s) and the
            # attention kernels address [B, S, h, d] views of the [S, B, ...] memory through their TMA strides - no transpose copies
            s, b = qkv.shape[0], qkv.shape[1]
            pid = _seq_major_positions(s, b, _raw(qkv).device)
            qkv = KR.apply_rope_packed(qkv, cos, sin, nh + nkv, total, hd, pid, neox=True)   # in place on the GEMM output (explicit positions)
            out = KAT.attention_packed(_raw(qkv).view(s, b, total, hd), nh, nkv, True, None, seq_major=True)   # [S, B, nh, hd]
            return self.o_proj(_w(_raw(out).reshape(s, b, nh * hd)))
        if cfg.sequence_parallel and self.mp > 1:   # [S, B, *] -> [B, S, *]
            qkv = qkv.transpose([1, 0, 2]).contiguous()
        b, s = qkv.shape[0], qkv.shape[1]
        qkv = KR.apply_rope_packed(qkv, cos, sin, nh + nkv, total, hd, position_ids, neox=True)
        out = KAT.attention_packed(_raw(qkv).view(b, s, total, hd), nh, nkv, True, None)   # [B, S, nh, hd]; q/k/v read in place
        out = _raw(out).reshape(b, s, nh * hd)
        if cfg.sequence_parallel and self.mp > 1:
            out = out.transpose(0, 1).contiguous()
        return self.o_proj(_w(out))


class LlamaMLP(nn.Layer):
    def __init__(self, config):
        super().__init__()
        mp = _mp_degree()
        h, f = config.hidden_size, config.intermediate_size
        std = config.initializer_range
        wattr = nn.ParamAttr(initializer=I.Normal(0.0, std))
        dattr = nn.ParamAttr(initializer=I.Normal(0.0, std / math.sqrt(2 * config.num_hidden_layers)))
        # fused gate|up projection -> packed SwiGLU
        if mp > 1:
            Col = mpu.ColumnSequenceParallelLinear if config.sequence_parallel else mpu.ColumnParallelLinear
            Row = mpu.RowSequenceParallelLinear if config.sequence_parallel else mpu.RowParallelLinear
            self.gate_up_proj = Col(h, 2 * f, weight_attr=wattr, has_bias=False, gather_output=False)
            self.down_proj = Row(f, h, weight_attr=dattr, has_bias=False, input_is_parallel=True)
        else:
            self.gate_up_proj = nn.Linear(h, 2 * f, weight_attr=wattr, bias_attr=False)
            self.down_proj = nn.Linear(f, h, weight_attr=dattr, bias_attr=False)

    def forward(self, x):
        return self.down_proj(KA.swiglu(self.gate_up_proj(x)))


class LlamaDecoderLayer(nn.Layer):
    def __init__(self, config, layer_idx=0):
        super().__init__()
        self.config, self.layer_idx = config, layer_idx
        self.input_layernorm = LlamaRMSNorm(config)
        self.self_attn = LlamaAttention(config)
        self.post_attention_layernorm = LlamaRMSNorm(config)
        self.mlp = LlamaMLP(config)

    def _forward(self, h, cos, sin, position_ids=None):
        if self._lean():
            return self._forward_lean(h, cos, sin, position_ids)
        x = self.input_layernorm(h)
        a = self.self_attn(x, cos, sin, position_ids)
        x, h = self.post_attention_layernorm(a, residual=h)     # fused: h = h + a ; x = rmsnorm(h)
        return h + self.mlp(x)

    def _lean(self):
        # single-GPU (no tensor parallel) CUDA training: norm->linear and swiglu->linear run as memory-lean fused autograd nodes
        return self.self_attn.mp == 1 and self.training and self.input_layernorm.weight.is_cuda and self.config.lean_activations

    def _forward_lean(self, h, cos, sin, position_ids=None):
        from ..kernels import fused_blocks as FB

        at, mlp = self.self_attn, self.mlp
        qkv = FB.norm_linear(h, self.input_layernorm.weight, at.qkv_proj.weight, self.input_layernorm.eps)
        a = at.attend(qkv, cos, sin, position_ids)
        gu, h = FB.norm_linear(a, self.post_attention_layernorm.weight, mlp.gate_up_proj.weight, self.post_attention_layernorm.eps, residual=h)
        return h + FB.swiglu_linear(gu, mlp.down_proj.weight)

    def forward(self, h, cos=None, sin=None, position_ids=None):
        if cos is None:
            cos, sin = rope_cache(self.config, h.device)
        if self.config.recompute and self.training and torch.is_grad_enabled() and not getattr(self, "_skip_recompute", False):
            return recompute(self._forward, h, cos, sin, position_ids)
        return self._forward(h, cos, sin, position_ids)


_pid_cache = {}


def _seq_major_positions(s, b, device):
    key = (s, b, str(device))
    t = _pid_cache.get(key)
    if t is None:
        if len(_pid_cache) > 16:
            _pid_cache.clear()
        t = _pid_cache[key] = torch.arange(s, device=device, dtype=torch.int64).repeat_interleave(b).reshape(1, s * b)
    return t


def rope_cache(config, device):
    cos, sin = KR.rope_tables(config.max_position_embeddings, config.head_dim, config.rope_theta, device)
    return cos, sin


class LlamaEmbedding(nn.Layer):
    def __init__(self, config):
        super().__init__()
        self.config = config
        attr = nn.ParamAttr(initializer=I.Normal(0.0, config.initializer_range))
        if _mp_degree() > 1:
            self.embed_tokens = mpu.VocabParallelEmbedding(config.vocab_size, config.hidden_size, weight_attr=attr)
        else:
            self.embed_tokens = nn.Embedding(config.vocab_size, config.hidden_size, weight_attr=attr)

    def forward(self, input_ids):
        h = self.embed_tokens(input_ids)
        if self.config.sequence_parallel and _mp_degree() > 1:
            h = _w(mpu.ScatterOp.apply(_raw(h).transpose(0, 1).contiguous()))   # [B,S,H] -> [S/p, B, H]
        return h


class LlamaLMHead(nn.Layer):
    """Final norm + (vocab-parallel) output projection."""

    def __init__(self, config):
        super().__init__()
        self.config = config
        self.norm = LlamaRMSNorm(config)
        mp = _mp_degree()
        self.mp = mp
        vocab_local = config.vocab_size // mp
        from ..distributed.fleet.random import get_rng_state_tracker

        with get_rng_state_tracker().rng_state():
            self.weight = self.create_parameter([config.hidden_size, vocab_local], default_initializer=I.Normal(0.0, config.initializer_range))
        self.weight.is_distributed = mp > 1
        if mp > 1:
            hcg = topo.get_hybrid_communicate_group()
            mpu._mark_dist_shard(self.weight, 1, hcg.get_model_parallel_rank(), mp)

    def forward(self, h):
        h = self.norm(h)
        if self.config.sequence_parallel and self.mp > 1:
            h = _w(mpu.AllGatherOp.apply(_raw(h)))                  # [S, B, H]
            h = h.transpose([1, 0, 2])
        elif self.mp > 1:
            h = mpu._c_identity(h)
        return F.linear(h, self.weight)                              # [B, S, V/mp] (kept vocab-parallel for the loss)


class LlamaPretrainingCriterion(nn.Layer):
    """Mean token cross-entropy on (vocab-parallel) logits; fused kernel."""

    def __init__(self, config=None, ignore_index=-100):
        super().__init__()
        self.ignore_index = ignore_index
        self.vocab_size = config.vocab_size if config is not None else None

    def forward(self, logits, labels):
        lg, lab = _raw(logits), _raw(labels).reshape(-1)
        v = lg.shape[-1]
        mp = _mp_degree()
        if self.vocab_size is not None and v == self.vocab_size:
            mp = 1  # logits carry the full vocabulary (dense model, or gathered): plain fused CE
        if mp > 1:
            hcg = topo.get_hybrid_communicate_group()
            grp = hcg.get_model_parallel_group()
            loss = KL.vocab_parallel_cross_entropy(lg.reshape(-1, v), lab, hcg.get_model_parallel_rank() * v, grp.pg, self.ignore_index)
        else:
            loss = KL.softmax_cross_entropy(lg.reshape(-1, v), lab, self.ignore_index, inplace_backward=True)
        loss = _raw(loss)
        valid = (lab != self.ignore_index).sum().clamp(min=1)
        return _w(loss.sum() / valid.to(loss.dtype))


class LlamaModel(nn.Layer):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.embedding = LlamaEmbedding(config)
        self.layers = nn.LayerList([LlamaDecoderLayer(config, i) for i in range(config.num_hidden_layers)])
        for l in list(self.layers)[len(self.layers) - config.recompute_skip_layers:] if config.recompute_skip_layers else []:
            l._skip_recompute = True

    def forward(self, input_ids, position_ids=None):
        h = self.embedding(input_ids)
        cos, sin = rope_cache(self.config, h.device)
        for layer in self.layers:
            h = layer(h, cos, sin, position_ids)
        return h


class LlamaForCausalLM(nn.Layer):
    def __init__(self, config):
        super().__init__()
        self.config = config
        self.llama = LlamaModel(config)
        self.lm_head = LlamaLMHead(config)
        self.criterion = LlamaPretrainingCriterion(config)

    def forward(self, input_ids, labels=None, position_ids=None):
        h = self.llama(input_ids, position_ids)
        logits = self.lm_head(h)
        if labels is None:
            return logits
        return self.criterion(logits, labels)

    def num_parameters(self):
        return sum(p.numel() for p in self.parameters())


def pipeline_layer_descs(config):
    """LayerDesc list for fleet.meta_parallel.PipelineLayer (embedding | decoder x L | head)."""
    from ..distributed.fleet.pipeline import LayerDesc

    descs = [LayerDesc(LlamaEmbedding, config)]
    descs += [LayerDesc(LlamaDecoderLayer, config, i) for i in range(config.num_hidden_layers)]
    descs.append(LayerDesc(LlamaLMHead, config))
    return descs
