"""CINN-role tensor compiler: fuses chains of elementwise / broadcast / last-axis-reduction ops of a recorded program into generated
CUDA kernels for sm_90a.

    fn = paddle.jit.to_static(f, backend="CINN")          # no-grad calls run the fused program
    prog2, report = paddle_b200.cinn.compile_program(program, fetch_list)      # static.Program -> static.Program

Pipeline (reference: paddle/cinn - decompose, op fusion, group schedule, CodeGenCUDA_Dev, runtime module):
  recorded static.Program --translate_to_pir--> SSA IR --pir passes / DRR patterns--> `fusion.fuse` (groups; composite ops such as softmax,
  gelu, silu, mean are decomposed to primitives on the way in: `expr.Frontend`) --`codegen`--> CUDA C++ (flat 4-wide elementwise kernels;
  warp-per-row / CTA-per-row reduction kernels) --`runtime`--> nvcc -gencode arch=compute_90a,code=sm_90a, cached in-tree, launched on
  the current stream through ctypes.  The same bodies are emitted as plain C++ for the host, which is how tests/test_cinn_cpu.py runs the
  compiler end to end without a GPU.  GEMM-shaped and attention ops are NOT generated: they stay on the hand-written wgmma kernels.
"""
from __future__ import annotations

from . import codegen, expr, fusion, runtime  # noqa: F401
from .expr import Unsupported  # noqa: F401
from .fusion import FusionResult, fuse  # noqa: F401
from .runtime import CompileError, FusedKernel, clear_cache, stats  # noqa: F401


def is_available():
    from ..pir import core_available

    return core_available()


def compile_program(program, fetch_list=None, min_ops=2, precompile=False, return_report=True):
    """static.Program -> optimised static.Program whose fusible chains run as generated kernels."""
    from .. import pir

    new = pir.optimize(program, fetch_list, cinn={"min_ops": min_ops, "precompile": precompile})
    return (new, new._cinn_report) if return_report else new


def nvcc_check(kernel):
    """Build the CUDA object of a FusedKernel without launching it (cross-compiles on a machine without a GPU).  Returns the .so path."""
    return runtime.compile_source(kernel.source("cuda"), "cuda")
