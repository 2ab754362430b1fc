"""NVLS (NVLink SHARP multicast) collectives: the NVSwitch adds / replicates, the kernels only issue `multimem.ld_reduce` / `multimem.st`.

Plumbing is torch.distributed._symmetric_memory (multicast object creation, binding and handle exchange between the processes);
the device code is ours (csrc/comm/nvls_collectives.cu).  A context owns ONE symmetric staging buffer per group; tensors are copied in and
out of it (the gradient arenas of parallel/arena.py can be placed inside it to skip the copies: `NvlsContext.tensor`).

Opt-in: FLAGS_b200_nvls (default off).  STATUS: the kernels are compiled for sm_90a (SASS shows LDGMC / multicast stores) but this path has
NOT run on hardware yet; tests/test_distributed_gpu.py::test_nvls_* is the 2-GPU check.  Without multicast support (no NVSwitch, driver
without fabric manager) `context_for` returns None and callers keep the peer-memory two-shot (parallel/symm.py) or NCCL.
Parity (role): NCCL's NVLS algorithm behind ProcessGroupNCCL all-reduce / reduce-scatter / all-gather."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

_contexts = {}
_PAD_TAIL = 256          # our barrier words: the last 256 bytes of every signal pad (2 slots x 8 ranks x 4 B = 64 B used)


def _pg(group):
    pg = getattr(group, "pg", group)
    return pg if pg is not None else dist.group.WORLD


def enabled():
    from ..framework.flags import flag

    return bool(flag("FLAGS_b200_nvls", False)) and torch.cuda.is_available() and dist.is_available() and dist.is_initialized()


def context_for(group, nbytes=None):
    """NvlsContext of the group, or None when NVLS cannot be used here."""
    if not enabled():
        return None
    pg = _pg(group)
    key = id(pg)
    if key not in _contexts:
        try:
            _contexts[key] = NvlsContext(pg, nbytes or int(os.environ.get("B200_NVLS_BUFFER_MB", "512")) << 20)
        except Exception as e:  # noqa: BLE001
            import warnings

            warnings.warn(f"paddle_b200: NVLS setup failed ({type(e).__name__}: {e}); using the peer-memory / NCCL collectives")
            _contexts[key] = None
    return _contexts[key]


class NvlsContext:
    def __init__(self, pg, nbytes):
        import torch.distributed._symmetric_memory as symm

        from .._build import ext

        self.ext = ext()
        if not hasattr(self.ext, "nvls_allreduce"):
            raise RuntimeError("extension built without the NVLS kernels")
        self.pg, self.world, self.rank = pg, dist.get_world_size(pg), dist.get_rank(pg)
        if self.world > 8:
            raise RuntimeError("NVLS kernels address at most 8 ranks (one NVSwitch domain)")
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.nbytes = (int(nbytes) + 4095) // 4096 * 4096
        self.buf = symm.empty(self.nbytes, dtype=torch.uint8, device=self.dev)
        self.h = symm.rendezvous(self.buf, pg)
        self.mc = int(self.h.multicast_ptr)
        if self.mc == 0:
            raise RuntimeError("the symmetric-memory handle has no multicast pointer (no NVLS on this system)")
        self.pads = [int(p) for p in self.h.signal_pad_ptrs]
        self.pad_off = int(self.h.signal_pad_size) - _PAD_TAIL
        if self.pad_off < 1024:
            raise RuntimeError("signal pad too small")
        self.local = int(self.buf.data_ptr())
        self.counter = torch.zeros(16, dtype=torch.int32, device=self.dev)
        self.epoch = 0
        # our barrier words must be zero on every rank before the first epoch is published
        self.h.barrier(0)
        self.h.get_signal_pad(self.rank, (_PAD_TAIL // 4,), torch.int32, self.pad_off // 4).zero_()
        torch.cuda.current_stream().synchronize()
        self.h.barrier(0)

    def _next(self):
        self.epoch += 1
        return self.epoch

    def tensor(self, offset, shape, dtype):
        """View of the staging buffer (16-byte aligned offset): data written here needs no copy-in."""
        n = 1
        for s in shape:
            n *= int(s)
        nb = n * torch.empty(0, dtype=dtype).element_size()
        if offset % 16 or offset + nb > self.nbytes:
            raise ValueError("offset / size outside the NVLS buffer")
        return self.buf[offset: offset + nb].view(dtype).view(*shape)

    def owns(self, t):
        return self.local <= t.data_ptr() and t.data_ptr() + t.numel() * t.element_size() <= self.local + self.nbytes

    @staticmethod
    def supports(t):
        return t.is_cuda and t.is_contiguous() and t.dtype in (torch.float32, torch.bfloat16, torch.float16) and (t.numel() * t.element_size()) % 16 == 0

    # ---- collectives ---------------------------------------------------------------------------------------------------------------------
    def all_reduce_(self, t):
        """In-place sum over the group.  Tensors inside the buffer are reduced where they are; others go through the front of the buffer
        in windows."""
        flat = t.reshape(-1)
        if self.owns(flat):
            self.ext.nvls_allreduce(self.pads, self.pad_off, self.mc, self.local, flat.data_ptr() - self.local, flat.numel(), flat.dtype, self.rank, self._next(),
                                    self.counter)
            return t
        es = flat.element_size()
        per = self.nbytes // es // (16 // es) * (16 // es)
        for lo in range(0, flat.numel(), per):
            hi = min(flat.numel(), lo + per)
            stage = self.tensor(0, (hi - lo,), flat.dtype)
            stage.copy_(flat[lo:hi])
            self.ext.nvls_allreduce(self.pads, self.pad_off, self.mc, self.local, 0, hi - lo, flat.dtype, self.rank, self._next(), self.counter)
            flat[lo:hi].copy_(stage)
        return t

    def reduce_scatter(self, out, inp):
        """out (n / world elements) = slice `rank` of sum over ranks of inp (n elements)."""
        flat = inp.reshape(-1)
        n, es = flat.numel(), flat.element_size()
        if n % self.world or (n // self.world * es) % 16 or n * es > self.nbytes:
            raise ValueError("reduce_scatter: the input must split into 16-byte aligned slices that fit the NVLS buffer")
        off = flat.data_ptr() - self.local if self.owns(flat) else 0
        if not self.owns(flat):
            self.tensor(0, (n,), flat.dtype).copy_(flat)
        self.ext.nvls_reduce_scatter(self.pads, self.pad_off, self.mc, self.local, off, out, n, self.rank, self._next(), self.counter)
        return out

    def all_gather(self, out, inp):
        """out (world * chunk) = concatenation over ranks of inp (chunk): every rank multicasts its chunk into slot `rank` of every replica."""
        chunk = inp.numel() * inp.element_size()
        if chunk % 16 or chunk * self.world > self.nbytes:
            raise ValueError("all_gather: chunks must be 16-byte multiples that fit the NVLS buffer")
        self.ext.nvls_allgather(self.pads, self.pad_off, self.mc, self.local, 0, inp.contiguous(), self.rank, self._next(), self.counter)
        out.reshape(-1).copy_(self.tensor(0, (out.numel(),), out.dtype))
        return out
