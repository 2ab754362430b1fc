"""int8 activations: the torch paths of paddle.matmul on int8, the per-token quantizer, the dequantising GEMM and llm_int8_linear against
float64 / int64 evaluations, and an llm.int8 model served by LLMEngine (CPU)."""
import copy

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models, nn
from paddle_b200.kernels import gemm_int8 as G8
from paddle_b200.nn import quant as Q


def _p(t):
    return t.as_subclass(paddle.Tensor)


def test_matmul_int8_is_exact_int32():
    a = paddle.to_tensor([[100, 100]], dtype="int8")
    b = paddle.to_tensor([[100], [100]], dtype="int8")
    out = paddle.matmul(a, b)
    assert out.dtype == torch.int32 and out.as_subclass(torch.Tensor).tolist() == [[20000]]
    g = torch.Generator().manual_seed(0)
    x = torch.randint(-128, 128, (3, 5, 40), generator=g, dtype=torch.int8)
    y = torch.randint(-128, 128, (3, 7, 40), generator=g, dtype=torch.int8)
    ref = torch.einsum("bmk,bnk->bmn", x.long(), y.long())
    assert torch.equal(paddle.matmul(_p(x), _p(y), transpose_y=True).as_subclass(torch.Tensor), ref.int())
    assert torch.equal(paddle.matmul(_p(x), _p(y.transpose(1, 2).contiguous())).as_subclass(torch.Tensor), ref.int())
    xt = x.transpose(1, 2).contiguous()
    assert torch.equal(paddle.matmul(_p(xt), _p(y), transpose_x=True, transpose_y=True).as_subclass(torch.Tensor), ref.int())
    full = torch.full((4, 2048), -128, dtype=torch.int8)                # the worst-case sum: 2048 * 128 * 128
    assert paddle.matmul(_p(full), _p(full), transpose_y=True).as_subclass(torch.Tensor).unique().tolist() == [2048 * 128 * 128]
    assert paddle.matmul(_p(torch.ones(3, 4)), _p(torch.ones(4, 2))).dtype == torch.float32    # other dtypes keep their path


def _quant_ref64(x, mask=None):
    xf = x.double()
    if mask is not None:
        xf = xf.masked_fill(mask, 0.0)
    s = xf.abs().amax(-1, keepdim=True).clamp(min=1e-8) / 127.0
    return s.reshape(-1)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_quantize_int8_rows(dtype):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(9, 64, generator=g) * 3).to(dtype)
    x[2] = 0                                                            # an all-zero row
    mask = torch.zeros(64, dtype=torch.bool)
    mask[[3, 17, 40]] = True
    for m in (None, mask):
        q, s = G8.quantize_int8_rows(x, m)
        assert q.dtype == torch.int8 and s.dtype == torch.float32 and s.shape == (9,)
        assert torch.allclose(s.double(), _quant_ref64(x, m), rtol=1e-6)
        assert (q[2] == 0).all() and torch.isfinite(s).all()
        if m is not None:
            assert (q[:, m] == 0).all()
        deq = q.double() * s.double().unsqueeze(1)
        xm = x.double() if m is None else x.double().masked_fill(m, 0.0)
        assert ((deq - xm).abs() <= s.double().unsqueeze(1) * 0.5 * (1 + 1e-6)).all()     # at most half a step from x
        assert q.abs().max() <= 127


def test_gemm_int8_dequant_torch_expression():
    g = torch.Generator().manual_seed(2)
    a = torch.randint(-128, 128, (5, 48), generator=g, dtype=torch.int8)
    b = torch.randint(-128, 128, (6, 48), generator=g, dtype=torch.int8)
    rs, cs, bias = torch.rand(5, generator=g), torch.rand(6, generator=g), torch.randn(6, generator=g)
    acc = a.long() @ b.long().t()
    assert torch.equal(G8.gemm_int8(a, b), acc.int())
    for out_dtype in (torch.float32, torch.bfloat16, torch.float16):
        for bb in (None, bias):
            y = G8.gemm_int8_dequant(a, b, rs, cs, bb, out_dtype)
            ref = acc.float() * rs.unsqueeze(1) * cs
            if bb is not None:
                ref = ref + bb
            assert y.dtype == out_dtype and torch.equal(y, ref.to(out_dtype))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_llm_int8_linear_torch_path_against_float64(dtype):
    g = torch.Generator().manual_seed(3)
    k, n = 64, 24
    x = torch.randn(2, 5, k, generator=g).to(dtype)
    x[..., [7, 30]] *= 40                                               # planted outlier columns
    w = torch.randn(k, n, generator=g) * 0.05
    bias = (torch.randn(n, generator=g) * 0.1).to(dtype)
    q, s = Q.weight_quantize(_p(w), algo="llm.int8")
    q, s = q.as_subclass(torch.Tensor), s.as_subclass(torch.Tensor)
    y = Q.llm_int8_linear(_p(x), _p(q), _p(bias), _p(s), threshold=6.0).as_subclass(torch.Tensor)
    assert y.shape == (2, 5, n) and y.dtype == dtype
    # float64 evaluation of the same decomposition
    x2 = x.reshape(-1, k).double()
    out = (x2.abs() > 6.0).any(0)
    assert out.tolist().count(True) == 2
    xi = x2.masked_fill(out, 0.0)
    sx = xi.abs().amax(-1, keepdim=True).clamp(min=1e-8) / 127.0
    xq = torch.round(xi / sx).clamp(-128, 127)
    wd = Q.weight_dequantize(_p(q), _p(s), "weight_only_int8", dtype).as_subclass(torch.Tensor).double()
    ref = (xq @ q.double().t()) * sx * s.double() + x2[:, out] @ wd[out] + bias.double()
    err = (y.reshape(-1, n).double() - ref).norm() / ref.norm()
    assert err < 1e-2, err
    # threshold inf: no outlier columns, the same as the dequantising GEMM with the bias in its epilogue
    yi = Q.llm_int8_linear(_p(x), _p(q), _p(bias), _p(s), threshold=float("inf")).as_subclass(torch.Tensor)
    xq2, sx2 = G8.quantize_int8_rows(x.reshape(-1, k))
    assert torch.equal(yi.reshape(-1, n), G8.gemm_int8_dequant(xq2, q, sx2, s, bias, dtype))


def _llama(seed=0, **kw):
    paddle.seed(seed)
    m = models.LlamaForCausalLM(models.llama_tiny(**{**dict(hidden_size=128, intermediate_size=256, num_attention_heads=4,
                                                             num_key_value_heads=2, vocab_size=256, max_position_embeddings=128), **kw}))
    m.eval()
    return m


def test_quantize_weights_llm_int8_layers_and_errors():
    from paddle_b200.models.weight_only import _targets

    m = models.quantize_weights(_llama(), "llm.int8", threshold=float("inf"))
    layers = [getattr(p, nm) for p, nm in _targets(m)]
    assert layers and all(isinstance(layer, models.LLMInt8Linear) for layer in layers)
    lin = layers[0]
    assert lin.quant_weight.dtype == torch.int8 and list(lin.quant_weight.shape) == [lin.out_features, lin.in_features]
    assert lin.weight_scale.dtype == torch.float32 and lin.threshold == float("inf")
    with pytest.raises(ValueError, match="already quantized"):
        models.quantize_weights(m, "llm.int8")
    with pytest.raises(ValueError, match="group_size"):
        models.quantize_weights(_llama(), "llm.int8", 128)
    with pytest.raises(ValueError, match="experts"):
        models.quantize_weights(models.MixtralForCausalLM(models.mixtral_tiny(vocab_size=256)), "llm.int8", experts=True)
    holder = _llama()
    holder.llama.layers[0].mlp.down_proj = nn.Linear(24, 128)
    with pytest.raises(ValueError, match="% 16"):
        models.quantize_weights(holder, "llm.int8")
    assert isinstance(holder.llama.layers[0].self_attn.qkv_proj, nn.Linear)    # nothing was replaced
    holder.llama.layers[0].self_attn.o_proj = object.__new__(nn.Layer)
    nn.Layer.__init__(holder.llama.layers[0].self_attn.o_proj)
    with pytest.raises(ValueError, match="nn.Linear"):
        models.quantize_weights(holder, "llm.int8")


@pytest.mark.parametrize("threshold", [float("inf"), 6.0])
def test_engine_serves_an_llm_int8_model(threshold):
    qm = models.quantize_weights(_llama(), "llm.int8", threshold=threshold)
    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(1, 256, (n,), generator=g).tolist() for n in (9, 33, 20)]
    eng = models.LLMEngine(qm, num_blocks=64, block_size=16)
    ids = [eng.add_request(p, 6) for p in prompts]
    res = eng.run_until_done()
    for i, p in zip(ids, prompts):
        out = models.generate(qm, torch.tensor([p]), max_new_tokens=6).as_subclass(torch.Tensor)[0, len(p):].tolist()
        assert res[i] == out
    eng = models.LLMEngine(qm, num_blocks=64, block_size=16, max_prefill_chunk=16)      # chunked prefill
    ids2 = [eng.add_request(p, 6) for p in prompts]
    res2 = eng.run_until_done()
    assert [res2[i] for i in ids2] == [res[i] for i in ids]
