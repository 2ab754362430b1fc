"""models.quantize_weights: weight-only int8 / int4 projection layers (`WeightOnlyLinear`) in Llama, Mixtral and GPT; greedy serving of a
quantised model through generate() and LLMEngine (mid-flight arrivals, chunked prefill, preemption, a quantised draft), engine logits
bit for bit against a 16-bit model holding the dequantised weights, and every documented error."""
import copy

import pytest
import torch

import paddle_b200 as paddle
from paddle_b200 import models, nn
from paddle_b200.nn import quant as Q

SPECS = [("weight_only_int8", -1), ("weight_only_int8", 64), ("weight_only_int4", -1), ("weight_only_int4", 128)]
NAMES = {"llama": ("qkv_proj", "o_proj", "gate_up_proj", "down_proj"), "mixtral": ("qkv_proj", "o_proj"), "gpt": ("qkv", "proj", "fc1", "fc2")}


def _model(kind, seed=0, **kw):
    paddle.seed(seed)
    if kind == "llama":
        m = models.LlamaForCausalLM(models.llama_tiny(**{**dict(hidden_size=128, intermediate_size=256, num_attention_heads=4,
                                                                 num_key_value_heads=2, vocab_size=256, max_position_embeddings=128), **kw}))
    elif kind == "mixtral":
        m = models.MixtralForCausalLM(models.mixtral_tiny(**{**dict(vocab_size=256), **kw}))
    else:
        m = models.GPTForCausalLM(models.gpt_tiny(**{**dict(vocab_size=256), **kw}))
        for blk in m.gpt.blocks:                                     # non-zero biases, so the bias path is exercised
            for lin in (blk.qkv, blk.proj, blk.fc1, blk.fc2):
                with torch.no_grad():
                    lin.bias.as_subclass(torch.Tensor).normal_(0, 0.02)
    m.eval()
    return m


def _targets(m):
    from paddle_b200.models.weight_only import _targets

    return _targets(m)


def _alone(m, prompt, n):
    out = models.generate(m, torch.tensor([prompt]), max_new_tokens=n).as_subclass(torch.Tensor)
    return out[0, len(prompt):].tolist()


def _prompts(vocab, lens, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, vocab, (n,), generator=g).tolist() for n in lens]


def _dequantized_copy(qm, ref):
    """A deep copy of the 16-bit model `ref` whose replaced Linear weights are the quantised model's dequantised weights."""
    d = copy.deepcopy(ref)
    for (qp, name), (dp, _) in zip(_targets(qm), _targets(d)):
        lin = getattr(dp, name)
        with torch.no_grad():
            lin.weight.as_subclass(torch.Tensor).copy_(getattr(qp, name).dequantized_weight(lin.weight.dtype).as_subclass(torch.Tensor))
    return d


@pytest.mark.parametrize("kind", ["llama", "mixtral", "gpt"])
def test_quantize_weights_replaces_exactly_the_projections(kind):
    m = _model(kind)
    before = {n for n, _ in m.named_parameters()}
    assert models.quantize_weights(m, "weight_only_int4", 64) is m
    replaced = {n for n, l in m.named_sublayers() if isinstance(l, models.WeightOnlyLinear)}
    assert {n.rsplit(".", 1)[1] for n in replaced} == set(NAMES[kind])
    assert len(replaced) == len(_targets(m))
    after = {n for n, _ in m.named_parameters()}
    assert before - after == {f"{r}.{p}" for r in replaced for p in ("weight", "bias") if f"{r}.{p}" in before}
    assert all(not isinstance(l, models.WeightOnlyLinear) for n, l in m.named_sublayers() if n not in replaced)
    if kind == "mixtral":                                            # the experts, router and LM head stay 16-bit
        assert any(".moe." in n for n in after) and "lm_head.weight" in after
    for r in replaced:
        layer = dict(m.named_sublayers())[r]
        assert layer.quant_weight.dtype == torch.int8 and layer.weight_scale.dtype == torch.float32
        assert {n for n, _ in layer.named_buffers()} >= {"quant_weight", "weight_scale"}


@pytest.mark.parametrize("algo,gs", SPECS)
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("shape", [(5, 128), (2, 3, 128)])
def test_weight_only_linear_layer_equals_linear_on_the_dequantized_weight(algo, gs, bias, shape):
    paddle.seed(1)
    lin = nn.Linear(128, 96, bias_attr=None if bias else False)
    if bias:
        with torch.no_grad():
            lin.bias.as_subclass(torch.Tensor).normal_()
    layer = models.WeightOnlyLinear(lin, algo, gs)
    assert layer.parameters() == []
    x = torch.randn(*shape).as_subclass(paddle.Tensor)
    w = Q.weight_dequantize(layer.quant_weight, layer.weight_scale, algo, torch.float32, gs)
    ref = nn.functional.linear(x, w, lin.bias if bias else None).as_subclass(torch.Tensor)
    out = layer(x).as_subclass(torch.Tensor)
    assert out.shape == (*shape[:-1], 96)
    assert torch.equal(out, ref)
    # the weight came from an fp32 copy: dequantised, it is within one quantisation step of the original
    step = layer.weight_scale.as_subclass(torch.Tensor).reshape(-1, 96)
    err = (w.as_subclass(torch.Tensor) - lin.weight.as_subclass(torch.Tensor)).abs().reshape(-1 if gs < 0 else 128 // gs, *(() if gs < 0 else (gs,)), 96)
    assert bool((err <= (step.unsqueeze(1) if gs > 0 else step) * 0.5 + 1e-7).all())


@pytest.mark.parametrize("kind", ["llama", "gpt", "mixtral"])
@pytest.mark.parametrize("algo,gs", [("weight_only_int8", -1), ("weight_only_int4", 128)])
def test_engine_greedy_tokens_equal_generate_on_the_quantized_model(kind, algo, gs):
    m = models.quantize_weights(_model(kind), algo, gs if kind != "gpt" or gs < 0 else 64)
    prompts = _prompts(256, (5, 17, 9, 3), seed=2)
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


@pytest.mark.parametrize("chunk", [3, 7])
def test_chunked_prefill_and_preemption_on_a_quantized_model(chunk):
    m = models.quantize_weights(_model("llama"), "weight_only_int4", 64)
    prompts = _prompts(256, (13, 22, 9), seed=3)
    news = [9, 7, 11]
    eng = models.LLMEngine(m, num_blocks=12, block_size=4, max_batch_tokens=12, max_prefill_chunk=chunk)   # too few blocks for all three
    ids = [eng.add_request(p, n) for p, n in zip(prompts, news)]
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n), (i, res[i])
    assert eng.stats["preemptions"] > 0
    assert eng.alloc.num_free() == 12


@pytest.mark.parametrize("kind", ["llama", "gpt"])
def test_engine_logits_equal_a_model_with_the_dequantized_weights(kind):
    ref = _model(kind)
    qm = models.quantize_weights(copy.deepcopy(ref), "weight_only_int4", 64)
    d = _dequantized_copy(qm, ref)
    prompts = _prompts(256, (11, 4, 19), seed=4)

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


def test_quantized_draft_keeps_the_16bit_target_tokens():
    m = _model("llama")
    d = models.quantize_weights(_model("llama", seed=5, num_hidden_layers=1), "weight_only_int4", 128)
    prompts = _prompts(256, (5, 17, 9), seed=6)
    news = [9, 6, 11]
    eng = models.LLMEngine(m, num_blocks=64, block_size=4, draft_model=d, num_speculative_tokens=3)
    ids = [eng.add_request(p, n) for p, n in zip(prompts, news)]
    res = eng.run_until_done()
    for i, p, n in zip(ids, prompts, news):
        assert res[i] == _alone(m, p, n)
    assert eng.stats["draft_tokens"] > 0


def test_quantized_model_forward_and_kv_calibration():
    for kind in ("llama", "gpt", "mixtral"):
        ref = _model(kind)
        qm = models.quantize_weights(copy.deepcopy(ref), "weight_only_int8", 64)
        ids = torch.tensor(_prompts(256, (7,), seed=7))
        out = qm(ids.as_subclass(paddle.Tensor)).as_subclass(torch.Tensor)
        assert torch.equal(out, _dequantized_copy(qm, ref)(ids.as_subclass(paddle.Tensor)).as_subclass(torch.Tensor))
    qm = models.quantize_weights(_model("llama"), "weight_only_int4", -1)
    absmax = models.calibrate_kv_cache(qm, _prompts(256, (9, 5), seed=8), block_size=4)
    assert bool((absmax.as_subclass(torch.Tensor) > 0).all())


def test_errors():
    with pytest.raises(ValueError, match="algo"):
        models.quantize_weights(_model("llama"), "weight_only_int2")
    with pytest.raises(ValueError, match="group_size"):
        models.quantize_weights(_model("llama"), "weight_only_int8", 32)
    with pytest.raises(ValueError, match="not a multiple of group_size"):
        models.quantize_weights(_model("llama", hidden_size=192, intermediate_size=256), "weight_only_int8", 128)
    holder = _model("gpt", hidden_size=64, intermediate_size=128, num_attention_heads=4)
    holder.gpt.blocks[0].fc2 = nn.Linear(7, 64)                      # an odd fan-in
    with pytest.raises(ValueError, match="odd"):
        models.quantize_weights(holder, "weight_only_int4")
    assert isinstance(holder.gpt.blocks[0].qkv, nn.Linear)           # nothing was replaced
    m = models.quantize_weights(_model("llama"), "weight_only_int8")
    with pytest.raises(ValueError, match="already quantized"):
        models.quantize_weights(m, "weight_only_int4")
