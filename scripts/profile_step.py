"""Per-kernel device-time breakdown of one training step of the flagship configuration (torch.profiler, CUDA activities).

Defaults to what `bench.py --gpus 1` runs: Llama-2-7B, full recompute, one 4096-token sequence per micro-batch, 4 micro-batches per
optimizer step, AdamW with fp32 master weights and bf16 moments over the flat gradient arena. Take it in a run of its own: tracing
slows the host, so the step time printed here is not the benchmark's.

  python scripts/profile_step.py [--layers N] [--micro-batches K] [--no-recompute] [--rows R]
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import paddle_b200 as paddle  # noqa: E402
from paddle_b200.models import llama as L  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--layers", type=int, default=0, help="decoder layers (default: all 32 of Llama-2-7B)")
ap.add_argument("--micro-batches", type=int, default=4)
ap.add_argument("--seq", type=int, default=4096)
ap.add_argument("--no-recompute", action="store_true")
ap.add_argument("--rows", type=int, default=30, help="rows of the kernel table")
args = ap.parse_args()

os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")
paddle.set_device("gpu:0")
paddle.set_default_dtype("bfloat16")
paddle.seed(1234)
cfg = L.llama2_7b(recompute=not args.no_recompute)
if args.layers:
    cfg.num_hidden_layers = args.layers
cfg.max_position_embeddings = args.seq
m = L.LlamaForCausalLM(cfg)
opt = paddle.optimizer.AdamW(1e-5, beta1=0.9, beta2=0.95, epsilon=1e-8, parameters=m.parameters(), weight_decay=0.1, multi_precision=True,
                             moment_dtype="bfloat16", grad_clip=paddle.nn.ClipGradByGlobalNorm(1.0))
opt.enable_flat_arena()
ids = torch.randint(0, cfg.vocab_size, (args.micro_batches, args.seq + 1), device="cuda").as_subclass(paddle.Tensor)


def step():
    for i in range(args.micro_batches):
        loss = m(ids[i:i + 1, :-1], ids[i:i + 1, 1:]) / args.micro_batches
        loss.backward()
    opt.step()
    opt.clear_grad()


for _ in range(2):
    step()
torch.cuda.synchronize()
s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s.record()
step()
e.record()
torch.cuda.synchronize()
print(f"step ms (profiler off) {s.elapsed_time(e):.1f}  layers={cfg.num_hidden_layers} micro_batches={args.micro_batches} seq={args.seq} "
      f"recompute={not args.no_recompute}", flush=True)
from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    step()
    torch.cuda.synchronize()
print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=args.rows, max_name_column_width=90))
