"""Global flags. Parity: paddle/common/flags.cc, python/paddle/base/framework.py:set_flags."""
from __future__ import annotations

import os

_FLAGS = {
    "FLAGS_check_nan_inf": False,
    "FLAGS_cudnn_deterministic": False,
    "FLAGS_use_fused_kernels": True,       # route nn/functional hot ops to the sm_90a kernels
    "FLAGS_b200_sync_debug": False,        # serialise side streams (race triage)
    "FLAGS_b200_p2p_collectives": True,    # fused compute+collective kernels over peer memory
    "FLAGS_b200_gemm_backend": "tcgen05",  # "tcgen05" | "cublas"
    "FLAGS_b200_nvls": False,              # all-reduce through NVSwitch multicast (parallel/nvls.py, multimem.ld_reduce / st); not yet run on hardware
    "FLAGS_b200_decode_kernel": False,     # models.generation: decode steps attend through csrc/decode_attention.cu (CUDA, head_dim 128 or 64, fp16 / bf16)
    "FLAGS_use_cinn": False,               # pir.optimize: fuse elementwise / reduction chains into generated sm_90a kernels (paddle_b200.cinn)
    "FLAGS_enable_pir_api": False,         # static Executor: run programs through the native IR pass pipeline (paddle_b200.pir) before replay
    "FLAGS_b200_fp8_block_scaled": False,  # with FLAGS_b200_fp8_linear: OCP MX scaling (one E8M0 scale per 32 k, applied per k-block in the fp8 GEMM) instead of per-tensor
    "FLAGS_b200_fp8_linear": False,        # nn.Linear / F.linear run as fp8 wgmma GEMMs (per-tensor scaling, e4m3 fwd / e5m2 grads)
    "FLAGS_b200_pp_mailbox": True,         # pipeline p2p through the peer-memory mailbox (copy engine + flag) instead of NCCL send/recv
    "FLAGS_b200_fused_wgrad": True,        # weight-gradient GEMMs accumulate straight into the flat gradient arena (kernels/wgrad.py)
    "FLAGS_b200_split_master_weights": True,   # bf16 arenas keep fp32 master weights as bf16 parameter + int16 residual (4 B instead of 6 B per parameter)
    "FLAGS_b200_to_static_train_graph": True,  # to_static captures training calls (forward + backward CUDA graphs) after two eager warm-ups
    "FLAGS_b200_moe_grouped_gemm": True,       # MoE experts run as grouped wgmma GEMMs with device-side routing
    "FLAGS_b200_flash_attention": True,    # wgmma flash-attention forward (csrc/attention_sm100.cu)
    "FLAGS_embedding_deterministic": 0,
    "FLAGS_eager_delete_tensor_gb": 0.0,
    "FLAGS_fraction_of_gpu_memory_to_use": 0.92,
    "FLAGS_allocator_strategy": "auto_growth",
    "FLAGS_b200_native_allocator": False,   # environment, at import: all CUDA memory through csrc/runtime/allocator.cpp instead of the torch caching allocator
    "FLAGS_enable_async_trace": False,
    "FLAGS_sync_nccl_allreduce": False,
    "FLAGS_max_inplace_grad_add": 0,
}


def _coerce(old, v):
    if isinstance(old, bool):
        return v if isinstance(v, bool) else str(v).lower() in ("1", "true", "yes", "on")
    if isinstance(old, int):
        return int(v)
    if isinstance(old, float):
        return float(v)
    return v


for _k in list(_FLAGS):
    if _k in os.environ:
        _FLAGS[_k] = _coerce(_FLAGS[_k], os.environ[_k])


def set_flags(flags: dict):
    for k, v in flags.items():
        _FLAGS[k] = _coerce(_FLAGS[k], v) if k in _FLAGS else v
        if k == "FLAGS_cudnn_deterministic":
            _apply_deterministic(bool(_FLAGS[k]))


def _apply_deterministic(on):
    """FLAGS_cudnn_deterministic reaches the hand-written kernels too: order-dependent reductions (the dQ bulk-reduce of the attention
    backward) take a fixed order; PyTorch's own switch covers the library kernels."""
    import torch

    try:
        torch.backends.cudnn.deterministic = bool(on)
    except Exception:  # noqa: BLE001
        pass
    try:
        from .._build import load

        m = load()
        if m is not None and hasattr(m, "set_deterministic"):
            m.set_deterministic(bool(on))
    except Exception:  # noqa: BLE001
        pass


def get_flags(names):
    if isinstance(names, str):
        names = [names]
    return {n: _FLAGS[n] for n in names}


def flag(name, default=None):
    return _FLAGS.get(name, default)


if _FLAGS.get("FLAGS_cudnn_deterministic"):
    _apply_deterministic(True)
