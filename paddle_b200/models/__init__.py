"""Model zoo for the BASELINE.json configs (Llama-2, GPT-3, Mixtral-MoE, ResNet-50, MNIST MLP)."""
from .llama import LlamaConfig, LlamaDecoderLayer, LlamaForCausalLM, LlamaModel, LlamaPretrainingCriterion, llama2_13b, llama_tiny, mistral_7b, tinyllama_1b  # noqa: F401
from .gpt import GPTConfig, GPTForCausalLM, GPTModel, gpt3_1p3b, gpt3_6p7b, gpt_tiny  # noqa: F401,E402
from .mixtral import MixtralConfig, MixtralForCausalLM, mixtral_8x7b, mixtral_tiny  # noqa: F401,E402
from .mlp import MnistMLP  # noqa: F401,E402
from .generation import KVCache, LlamaGenerator, generate  # noqa: F401,E402
from .serving import BlockAllocator, LLMEngine, calibrate_kv_cache  # noqa: F401,E402
from .weight_only import LLMInt8Linear, WeightOnlyLinear, quantize_weights  # noqa: F401,E402


def resnet50(**kw):
    from ..vision.models import resnet50 as _r

    return _r(**kw)
