"""GPT-3 family (pre-LN decoder, learned positions, GELU MLP, biases). Parity (role): the GPT used by the reference's
GroupSharded / auto-parallel benchmarks (test/auto_parallel/get_gpt_model.py, PaddleNLP gpt modeling).
Hot ops: fused-QKV wgmma GEMM with bias epilogue, wgmma flash attention, fused LayerNorm, bias+GELU GEMM epilogue."""
from __future__ import annotations

from dataclasses import dataclass

import torch

from .. import nn
from ..distributed.fleet.recompute import recompute
from ..kernels import attention as KAT
from ..kernels import gemm as KG
from ..kernels import loss as KL
from ..nn import functional as F
from ..nn import initializer as I
from ..tensor import Tensor


@dataclass
class GPTConfig:
    vocab_size: int = 50304
    hidden_size: int = 4096
    num_hidden_layers: int = 32
    num_attention_heads: int = 32
    intermediate_size: int = 16384
    max_position_embeddings: int = 2048
    layer_norm_eps: float = 1e-5
    initializer_range: float = 0.02
    recompute: bool = False
    dropout: float = 0.0

    @property
    def head_dim(self):
        return self.hidden_size // self.num_attention_heads


def gpt3_6p7b(**kw):
    return GPTConfig(**kw)


def gpt3_1p3b(**kw):
    return GPTConfig(hidden_size=2048, num_hidden_layers=24, num_attention_heads=16, intermediate_size=8192, **kw)


def gpt_tiny(**kw):
    base = dict(vocab_size=512, hidden_size=128, num_hidden_layers=2, num_attention_heads=4, intermediate_size=512, max_position_embeddings=128)
    base.update(kw)
    return GPTConfig(**base)


def _raw(t):
    return t.as_subclass(torch.Tensor) if isinstance(t, torch.Tensor) and type(t) is not torch.Tensor else t


class GPTBlock(nn.Layer):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        h, std = cfg.hidden_size, cfg.initializer_range
        w = nn.ParamAttr(initializer=I.Normal(0.0, std))
        wo = nn.ParamAttr(initializer=I.Normal(0.0, std / (2 * cfg.num_hidden_layers) ** 0.5))
        self.ln1 = nn.LayerNorm(h, epsilon=cfg.layer_norm_eps)
        self.qkv = nn.Linear(h, 3 * h, weight_attr=w)
        self.proj = nn.Linear(h, h, weight_attr=wo)
        self.ln2 = nn.LayerNorm(h, epsilon=cfg.layer_norm_eps)
        self.fc1 = nn.Linear(h, cfg.intermediate_size, weight_attr=w)
        self.fc2 = nn.Linear(cfg.intermediate_size, h, weight_attr=wo)

    def _forward(self, x):
        cfg = self.cfg
        b, s, h = x.shape
        qkv = _raw(self.qkv(self.ln1(x))).view(b, s, 3, cfg.num_attention_heads, cfg.head_dim)
        a = KAT.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], None, 0.0, True, None)
        x = x + self.proj(_raw(a).reshape(b, s, h).as_subclass(Tensor))
        y = self.ln2(x)
        y = KG.gemm(_raw(y).reshape(-1, h), self.fc1.weight, self.fc1.bias, epilogue=2).reshape(b, s, -1) if _fused_ok(y) else F.gelu(self.fc1(y))
        return x + self.fc2(y if isinstance(y, Tensor) else y.as_subclass(Tensor))

    def forward(self, x):
        if self.cfg.recompute and self.training and torch.is_grad_enabled():
            return recompute(self._forward, x)
        return self._forward(x)


def _fused_ok(y):
    # the bias+GELU epilogue variant has no autograd wrapper: inference only
    return (not torch.is_grad_enabled()) and y.is_cuda and y.dtype in (torch.bfloat16, torch.float16)


class TiedEmbedding(nn.Embedding):
    """Token embedding that also serves as the (tied) output projection: `emb(h, project=True)` = h @ W^T.  Both uses go through
    this layer's __call__, so parameter-sharding wrappers (GroupSharded stage 3 gathers a layer's weights in its forward hooks)
    see the weight materialised for the LM head as well."""

    def forward(self, x, project=False):
        if project:
            return F.linear(x, self.weight.t())
        return super().forward(x)


class GPTModel(nn.Layer):
    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        attr = nn.ParamAttr(initializer=I.Normal(0.0, cfg.initializer_range))
        self.wte = TiedEmbedding(cfg.vocab_size, cfg.hidden_size, weight_attr=attr)
        self.wpe = nn.Embedding(cfg.max_position_embeddings, cfg.hidden_size, weight_attr=attr)
        self.blocks = nn.LayerList([GPTBlock(cfg) for _ in range(cfg.num_hidden_layers)])
        self.ln_f = nn.LayerNorm(cfg.hidden_size, epsilon=cfg.layer_norm_eps)

    def forward(self, input_ids):
        s = input_ids.shape[1]
        pos = torch.arange(s, device=input_ids.device).unsqueeze(0)
        x = self.wte(input_ids) + self.wpe(pos.as_subclass(Tensor))
        for blk in self.blocks:
            x = blk(x)
        return self.ln_f(x)


class GPTForCausalLM(nn.Layer):
    """LM head tied to the token embedding (as in GPT-3)."""

    def __init__(self, cfg):
        super().__init__()
        self.cfg = cfg
        self.gpt = GPTModel(cfg)

    def forward(self, input_ids, labels=None):
        h = self.gpt(input_ids)
        logits = self.gpt.wte(h, project=True)
        if labels is None:
            return logits
        v = logits.shape[-1]
        loss = _raw(KL.softmax_cross_entropy(_raw(logits).reshape(-1, v), _raw(labels).reshape(-1), -100, inplace_backward=True))
        valid = (_raw(labels).reshape(-1) != -100).sum().clamp(min=1)
        return (loss.sum() / valid.to(loss.dtype)).as_subclass(Tensor)
