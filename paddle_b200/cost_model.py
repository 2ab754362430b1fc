"""paddle.cost_model: analytic step-time model used by distributed.auto_tuner. Parity: python/paddle/cost_model/cost_model.py."""


class CostModel:
    def __init__(self, peaks=None):
        self.peaks = peaks or self._load_peaks()

    @staticmethod
    def _load_peaks():
        return {"hbm_gbs": 3350.0, "bf16_tflops_sustained": 989.0}   # NVIDIA's data sheet for the H100 SXM (HBM3, dense bf16); pass measured ones

    def gemm_ms(self, m, n, k, eff=0.68):   # median share of 989 TFLOP/s of the own GEMM on Llama-2-7B's shapes (DESIGN.md §4)
        return 2.0 * m * n * k / (self.peaks.get("bf16_tflops_sustained", 989.0) * 1e9 * eff)

    def mem_ms(self, nbytes, eff=0.8):
        return nbytes / (self.peaks.get("hbm_gbs", 3350.0) * 1e6 * eff)

    def allreduce_ms(self, nbytes, world, bus_gbs=450.0):   # NVLink 4 data sheet, one direction; not measured
        return 0.0 if world <= 1 else 2.0 * (world - 1) / world * nbytes / (bus_gbs * 1e6)

    def profile_measure(self, main_program=None, startup_program=None, device="gpu", fetch_cost_list=("time",), feed=None, fetch_list=None, repeat=5):
        """Run a static Program (or any zero-argument callable) `repeat` times and return measured costs:
        {"time": ms per run (CUDA events on GPU, perf_counter on CPU), "kernel_launches": own-kernel launches per run}."""
        import time

        import torch

        if callable(main_program):
            run = main_program
        else:
            from . import static

            exe = static.Executor()
            if startup_program is not None:
                exe.run(startup_program)
            run = lambda: exe.run(main_program, feed=feed or {}, fetch_list=fetch_list or [])  # noqa: E731
        run()
        from . import _build

        C = _build.load(required=False)
        l0 = C.launch_count() if C is not None else 0
        on_gpu = torch.cuda.is_available() and device != "cpu"
        if on_gpu:
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(repeat):
                run()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / repeat
        else:
            t0 = time.perf_counter()
            for _ in range(repeat):
                run()
            ms = (time.perf_counter() - t0) * 1e3 / repeat
        out = {"time": ms, "kernel_launches": ((C.launch_count() - l0) / repeat) if C is not None else 0}
        return {k: out[k] for k in out if k in fetch_cost_list or k == "time"}
