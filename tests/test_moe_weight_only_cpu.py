"""Weight-only int8 / int4 MoE experts on the CPU: fused_moe(quant_method=...) bit for bit against fused_moe("None") on the dequantised
weights, every documented ValueError, quantize_weights(..., experts=True) on Mixtral, and LLMEngine serving an expert-quantised Mixtral
(greedy tokens against generate(), logits against a 16-bit copy holding the dequantised weights)."""
import copy

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models
from paddle_b200.incubate.moe import ExpertFFN, WeightOnlyExpertFFN
from paddle_b200.incubate.nn import functional as IF
from paddle_b200.nn import quant as Q

SPECS = [("weight_only_int8", -1), ("weight_only_int8", 64), ("weight_only_int8", 128),
         ("weight_only_int4", -1), ("weight_only_int4", 64), ("weight_only_int4", 128)]


def _p(t):
    return t.as_subclass(paddle.Tensor)


def _stack(w, algo, gs):
    """Stacked weight_quantize outputs of w [E, K, N] and the dequantised float stack [E, K, N]."""
    qs = [Q.weight_quantize(_p(w[e]), algo=algo, group_size=gs) for e in range(w.shape[0])]
    q = torch.stack([q.as_subclass(torch.Tensor) for q, _ in qs])
    s = torch.stack([s.as_subclass(torch.Tensor) for _, s in qs])
    d = torch.stack([Q.weight_dequantize(qq, ss, algo, torch.float32, gs).as_subclass(torch.Tensor) for qq, ss in qs])
    return q, s, d


def _moe_inputs(seed, E=4, d=128, f=128, bias=False):
    g = torch.Generator().manual_seed(seed)
    gate = torch.randn(d, E, generator=g)
    w1 = torch.randn(E, d, 2 * f, generator=g) * 0.05
    w2 = torch.randn(E, f, d, generator=g) * 0.05
    b1 = torch.randn(E, 1, 2 * f, generator=g) * 0.1 if bias else None
    b2 = torch.randn(E, 1, d, generator=g) * 0.1 if bias else None
    return g, gate, w1, w2, b1, b2


@pytest.mark.parametrize("algo,gs", SPECS)
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("xshape", [(7, 128), (2, 5, 128)])
@pytest.mark.parametrize("view", ["nk", "kn"])
def test_fused_moe_quantized_equals_float_on_the_dequantized_weights(algo, gs, bias, xshape, view):
    g, gate, w1, w2, b1, b2 = _moe_inputs(SPECS.index((algo, gs)), bias=bias)
    x = torch.randn(*xshape, generator=g)
    q1, s1, d1 = _stack(w1, algo, gs)
    q2, s2, d2 = _stack(w2, algo, gs)
    if view == "kn":                                                 # the reference test's reshaped view of the same bytes
        q1 = q1.reshape(q1.shape[0], 128, -1)
        q2 = q2.reshape(q2.shape[0], 128, -1)
    kw = dict(moe_topk=2, norm_topk_prob=True)
    out = IF.fused_moe(_p(x), _p(gate), _p(q1), _p(q2), None if b1 is None else _p(b1), _p(s1), None if b2 is None else _p(b2), _p(s2),
                       quant_method=algo, **kw).as_subclass(torch.Tensor)
    ref = IF.fused_moe(_p(x), _p(gate), _p(d1), _p(d2), None if b1 is None else _p(b1), None, None if b2 is None else _p(b2), None,
                       quant_method="None", **kw).as_subclass(torch.Tensor)
    assert out.shape == x.shape
    assert torch.equal(out, ref)
    # scales of another float dtype are read as fp32
    out16 = IF.fused_moe(_p(x), _p(gate), _p(q1), _p(q2), None, _p(s1.double()), None, _p(s2.double()), quant_method=algo, **kw)
    ref16 = IF.fused_moe(_p(x), _p(gate), _p(d1), _p(d2), None, None, None, None, **kw)
    assert torch.equal(out16.as_subclass(torch.Tensor), ref16.as_subclass(torch.Tensor))


def test_fused_moe_errors():
    g, gate, w1, w2, _, _ = _moe_inputs(3)
    x = _p(torch.randn(4, 128, generator=g))
    q1, s1, d1 = _stack(w1, "weight_only_int8", 64)
    q2, s2, d2 = _stack(w2, "weight_only_int8", 64)
    P = [_p(t) for t in (gate, q1, q2, s1, s2)]
    with pytest.raises(ValueError, match="quant_method"):
        IF.fused_moe(x, P[0], P[1], P[2], None, P[3], None, P[4], quant_method="weight_only_int2")
    with pytest.raises(ValueError, match="needs ffn1_scale and ffn2_scale"):
        IF.fused_moe(x, P[0], P[1], P[2], None, None, None, P[4], quant_method="weight_only_int8")
    with pytest.raises(ValueError, match="only used with a weight-only"):
        IF.fused_moe(x, P[0], _p(d1), _p(d2), None, P[3], None, P[4], quant_method="None")
    with pytest.raises(ValueError, match="int8 expert weights need"):
        IF.fused_moe(x, P[0], P[1], P[2])
    with pytest.raises(ValueError, match="neither"):                 # 128 / 4 = 32 is not a group size
        IF.fused_moe(x, P[0], P[1], P[2], None, _p(torch.ones(4, 4, 256)), None, P[4], quant_method="weight_only_int8")
    with pytest.raises(ValueError, match="neither"):
        IF.fused_moe(x, P[0], P[1], P[2], None, _p(torch.ones(4 * 256)), None, P[4], quant_method="weight_only_int8")
    with pytest.raises(ValueError, match="neither"):                 # scales of 3 experts for a 4-expert router
        IF.fused_moe(x, P[0], P[1], P[2], None, _p(s1[:3]), None, P[4], quant_method="weight_only_int8")
    with pytest.raises(ValueError, match="int8 bytes"):              # int8 bytes read as int4: twice the bytes the shapes need
        IF.fused_moe(x, P[0], P[1], P[2], None, P[3], None, P[4], quant_method="weight_only_int4")
    with pytest.raises(ValueError, match="int8 bytes"):
        IF.fused_moe(x, P[0], _p(q1[:, :100]), P[2], None, P[3], None, P[4], quant_method="weight_only_int8")
    # float calls without scales are unchanged
    out = IF.fused_moe(x, P[0], _p(d1), _p(d2)).as_subclass(torch.Tensor)
    assert out.shape == (4, 128) and bool(torch.isfinite(out).all())


def _mixtral(seed=0, **kw):
    paddle.seed(seed)
    m = models.MixtralForCausalLM(models.mixtral_tiny(**{**dict(vocab_size=256), **kw}))
    m.eval()
    return m


@pytest.mark.parametrize("algo,gs", [("weight_only_int8", -1), ("weight_only_int4", 64), ("weight_only_int8", 128)])
def test_quantize_weights_experts(algo, gs):
    m = _mixtral()
    before = {n for n, _ in m.named_parameters()}
    assert models.quantize_weights(m, algo, gs, experts=True) is m
    after = {n for n, _ in m.named_parameters()}
    cfg = m.cfg
    E, d, f = cfg.num_local_experts, cfg.hidden_size, cfg.intermediate_size
    for i, layer in enumerate(m.layers):
        ex = layer.moe.experts
        assert isinstance(ex, WeightOnlyExpertFFN) and ex.num_expert == E
        assert isinstance(layer.self_attn.qkv_proj, models.WeightOnlyLinear) and isinstance(layer.self_attn.o_proj, models.WeightOnlyLinear)
        assert f"layers.{i}.moe.experts.w1" in before and f"layers.{i}.moe.experts.w1" not in after
        assert f"layers.{i}.moe.experts.w2" not in after
        assert f"layers.{i}.moe.gate.gate.weight" in after                    # the router stays 16-bit
        div = 2 if "int4" in algo else 1
        assert tuple(ex.quant_w1.shape) == (E, 2 * f, d // div) and tuple(ex.quant_w2.shape) == (E, d, f // div)
        assert ex.quant_w1.dtype == torch.int8 and ex.quant_w2.dtype == torch.int8
        assert ex.scale_w1.dtype == torch.float32 and ex.scale_w2.dtype == torch.float32
        assert tuple(ex.scale_w1.shape) == ((E, 2 * f) if gs < 0 else (E, d // gs, 2 * f))
        assert tuple(ex.scale_w2.shape) == ((E, d) if gs < 0 else (E, f // gs, d))
        assert {n for n, _ in ex.named_buffers()} == {"quant_w1", "scale_w1", "quant_w2", "scale_w2"}
        assert ex.parameters() == []
    assert not any(".experts." in n for n in after)
    # the default leaves the experts 16-bit
    m2 = models.quantize_weights(_mixtral(), algo, gs)
    assert all(isinstance(layer.moe.experts, ExpertFFN) for layer in m2.layers)


def test_quantize_weights_experts_errors():
    with pytest.raises(ValueError, match="no MoE experts"):
        paddle.seed(0)
        models.quantize_weights(models.LlamaForCausalLM(models.llama_tiny(hidden_size=128, intermediate_size=256, num_attention_heads=4,
                                                                         num_key_value_heads=2, vocab_size=256)), experts=True)
    m = _mixtral(intermediate_size=192)                                          # f = 192: not a multiple of 128
    with pytest.raises(ValueError, match="ffn2: fan-in 192"):
        models.quantize_weights(m, "weight_only_int8", 128, experts=True)
    assert isinstance(m.layers[0].self_attn.qkv_proj, paddle.nn.Linear)          # nothing was replaced
    assert isinstance(m.layers[0].moe.experts, ExpertFFN)
    m = _mixtral(intermediate_size=97, hidden_size=128)
    with pytest.raises(ValueError, match="odd"):
        models.quantize_weights(m, "weight_only_int4", -1, experts=True)
    m = _mixtral()
    m.layers[1].moe.world_size = 2                                               # an expert-parallel layer
    with pytest.raises(ValueError, match="expert-parallel"):
        models.quantize_weights(m, "weight_only_int8", experts=True)
    assert isinstance(m.layers[0].moe.experts, ExpertFFN)
    m = models.quantize_weights(_mixtral(), "weight_only_int8", experts=True)
    with pytest.raises(ValueError, match="already quantized"):
        models.quantize_weights(m, "weight_only_int8", experts=True)


def _alone(m, prompt, n):
    out = models.generate(m, torch.tensor([prompt]), max_new_tokens=n).as_subclass(torch.Tensor)
    return out[0, len(prompt):].tolist()


def _prompts(lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, 256, (n,), generator=g).tolist() for n in lens]


@pytest.mark.parametrize("algo,gs", [("weight_only_int8", -1), ("weight_only_int4", 128)])
def test_engine_greedy_tokens_equal_generate_on_an_expert_quantized_mixtral(algo, gs):
    m = models.quantize_weights(_mixtral(), algo, gs, experts=True)
    prompts = _prompts((5, 17, 9, 3), seed=2)
    news = [6, 4, 8, 5]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4)
    ids = [eng.add_request(prompts[0], news[0]), eng.add_request(prompts[1], news[1])]
    eng.step()
    ids.append(eng.add_request(prompts[2], news[2]))                 # arrives while the others decode
    eng.step()
    ids.append(eng.add_request(prompts[3], news[3]))
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n), (i, res[i])
    assert eng.alloc.num_free() == 64


def test_chunked_prefill_and_preemption_on_an_expert_quantized_mixtral():
    m = models.quantize_weights(_mixtral(), "weight_only_int4", 64, experts=True)
    prompts = _prompts((13, 22, 9), seed=3)
    news = [9, 7, 11]
    eng = models.LLMEngine(m, num_blocks=12, block_size=4, max_batch_tokens=12, max_prefill_chunk=5)
    ids = [eng.add_request(p, n) for p, n in zip(prompts, news)]
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n), (i, res[i])
    assert eng.stats["preemptions"] > 0
    assert eng.alloc.num_free() == 12


def _dequantized_copy(qm, ref):
    """A deep copy of the 16-bit Mixtral `ref` holding the quantised model's dequantised attention projections and experts."""
    from paddle_b200.models.weight_only import _targets

    d = copy.deepcopy(ref)
    with torch.no_grad():
        for (qp, name), (dp, _) in zip(_targets(qm), _targets(d)):
            lin = getattr(dp, name)
            lin.weight.as_subclass(torch.Tensor).copy_(getattr(qp, name).dequantized_weight(lin.weight.dtype).as_subclass(torch.Tensor))
        for ql, dl in zip(qm.layers, d.layers):
            w1, w2 = ql.moe.experts.dequantized(dl.moe.experts.w1.dtype)
            dl.moe.experts.w1.as_subclass(torch.Tensor).copy_(w1)
            dl.moe.experts.w2.as_subclass(torch.Tensor).copy_(w2)
    return d


def test_engine_logits_equal_a_model_with_the_dequantized_experts():
    ref = _mixtral()
    qm = models.quantize_weights(copy.deepcopy(ref), "weight_only_int4", 64, experts=True)
    d = _dequantized_copy(qm, ref)
    prompts = _prompts((11, 4, 19), seed=4)

    def serve(model):
        eng = models.LLMEngine(model, num_blocks=64, block_size=4, max_prefill_chunk=5)
        logits = []
        fwd = eng._forward

        def record(seqs, n_new, enc, dec):
            out = fwd(seqs, n_new, enc, dec)
            logits.append(out.clone())
            return out

        eng._forward = record
        ids = [eng.add_request(p, 6) for p in prompts]
        res = eng.run_until_done()
        return [res[i] for i in ids], logits

    toks, lq = serve(qm)
    toks_d, ld = serve(d)
    assert toks == toks_d
    assert len(lq) == len(ld)
    for a, b in zip(lq, ld):
        assert torch.equal(a, b)
