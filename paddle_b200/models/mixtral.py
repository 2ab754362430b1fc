"""Mixtral-style sparse MoE decoder (Llama attention + top-2 routed SwiGLU experts, expert parallel over a group).
Parity (role): PaddleNLP mixtral / the reference's MoELayer benchmarks (python/paddle/incubate/distributed/models/moe/).
Experts are stored stacked ([E_local, ...]) so the per-expert FFNs run as grouped wgmma GEMMs; tokens travel through the
expert-parallel all-to-all (incubate.moe.global_scatter / global_gather; peer-memory all-to-all kernel when available)."""
from __future__ import annotations

from dataclasses import dataclass

import torch

from .. import nn
from ..incubate.moe import ExpertFFN, MoELayer
from ..kernels import loss as KL
from ..nn import functional as F
from ..nn import initializer as I
from ..tensor import Tensor
from .llama import LlamaAttention, LlamaConfig, LlamaRMSNorm, rope_cache


@dataclass
class MixtralConfig(LlamaConfig):
    vocab_size: int = 32000
    hidden_size: int = 4096
    intermediate_size: int = 14336
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    num_local_experts: int = 8
    num_experts_per_tok: int = 2
    router_aux_loss_coef: float = 0.02
    rope_theta: float = 1e6


def mixtral_8x7b(**kw):
    return MixtralConfig(**kw)


def mixtral_tiny(**kw):
    base = dict(vocab_size=512, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                num_local_experts=4, max_position_embeddings=128)
    base.update(kw)
    return MixtralConfig(**base)


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


class MixtralDecoderLayer(nn.Layer):
    def __init__(self, cfg, moe_group=None):
        super().__init__()
        self.cfg = cfg
        ep = moe_group.nranks if moe_group is not None else 1
        assert cfg.num_local_experts % ep == 0, "experts must divide evenly over the expert-parallel group"
        self.input_layernorm = LlamaRMSNorm(cfg)
        self.self_attn = LlamaAttention(cfg)
        self.post_attention_layernorm = LlamaRMSNorm(cfg)
        experts = ExpertFFN(cfg.num_local_experts // ep, cfg.hidden_size, cfg.intermediate_size, activation="swiglu")
        self.moe = MoELayer(cfg.hidden_size, experts, gate={"type": "naive", "top_k": cfg.num_experts_per_tok}, moe_group=moe_group)

    def forward(self, h, cos, sin):
        a = self.self_attn(self.input_layernorm(h), cos, sin, None)
        x, h = self.post_attention_layernorm(a, residual=h)
        return h + self.moe(x)


class MixtralForCausalLM(nn.Layer):
    def __init__(self, cfg, moe_group=None):
        super().__init__()
        self.cfg = cfg
        attr = nn.ParamAttr(initializer=I.Normal(0.0, cfg.initializer_range))
        self.embed_tokens = nn.Embedding(cfg.vocab_size, cfg.hidden_size, weight_attr=attr)
        self.layers = nn.LayerList([MixtralDecoderLayer(cfg, moe_group) for _ in range(cfg.num_hidden_layers)])
        self.norm = LlamaRMSNorm(cfg)
        self.lm_head = nn.Linear(cfg.hidden_size, cfg.vocab_size, weight_attr=attr, bias_attr=False)

    def forward(self, input_ids, labels=None):
        h = self.embed_tokens(input_ids)
        cos, sin = rope_cache(self.cfg, h.device)
        for layer in self.layers:
            h = layer(h, cos, sin)
        logits = self.lm_head(self.norm(h))
        if labels is None:
            return logits
        v = logits.shape[-1]
        loss = _raw(KL.softmax_cross_entropy(_raw(logits).reshape(-1, v), _raw(labels).reshape(-1), -100, inplace_backward=True))
        valid = (_raw(labels).reshape(-1) != -100).sum().clamp(min=1)
        return (loss.sum() / valid.to(loss.dtype)).as_subclass(Tensor)
