"""Parallel-strategy auto tuner.

Parity: python/paddle/distributed/auto_tuner/{tuner.py (AutoTuner: search_once / add_cfg / resume), search.py (grid + dp-estimation search),
prune.py (named prune rules incl. history-based ones), recorder.py (HistoryRecorder: sorted csv, best cfg), memory_cost_model.py,
cost_model.py} and the `--auto_tuner_json` mode of `paddle.distributed.launch`.

Pieces: `SearchSpace` enumerates (dp, mp, pp, sharding degree + stage, micro-batch, vpp, recompute, pipeline schedule, sequence parallel) for a
transformer; named prune rules throw candidates out before anything runs (divisibility, memory model, dominated-by-history: a config that
ran out of memory prunes every config that needs at least as much); the time model ranks the rest (GEMM / attention FLOPs over the measured
sustained peak, mp collectives, pipeline bubble per schedule, dp / sharding gradient traffic, optimizer HBM pass); `Recorder` keeps the trial
history on disk (json lines, resumable); `AutoTuner.tune` runs trials through a user command (one subprocess per candidate, environment
variables carry the candidate) or a Python callable and stops after `max_trials` / `max_time_s`.
"""
from __future__ import annotations

import itertools
import json
import os
import subprocess
import time

from ..cost_model import CostModel

GB = float(2 ** 30)


def _divisors(n):
    return [d for d in range(1, n + 1) if n % d == 0]


# ------------------------------------------------------------------------------------------------ model description
class ModelSpec:
    """Decoder-only transformer (Llama / GPT family) - enough to count parameters, activations and FLOPs."""

    def __init__(self, hidden, layers, ffn, vocab, seq, heads=None, kv_heads=None, gated_ffn=True, moe_experts=0, moe_topk=2):
        self.hidden, self.layers, self.ffn, self.vocab, self.seq = int(hidden), int(layers), int(ffn), int(vocab), int(seq)
        self.heads = int(heads) if heads else max(1, self.hidden // 128)
        self.kv_heads = int(kv_heads) if kv_heads else self.heads
        self.gated_ffn, self.moe_experts, self.moe_topk = bool(gated_ffn), int(moe_experts), int(moe_topk)

    @property
    def attn_params(self):
        kv = self.hidden * self.kv_heads // self.heads
        return 2 * self.hidden * self.hidden + 2 * self.hidden * kv

    @property
    def ffn_params(self):
        per = (3 if self.gated_ffn else 2) * self.hidden * self.ffn
        return per * max(1, self.moe_experts)

    @property
    def layer_params(self):
        return self.attn_params + self.ffn_params + 2 * self.hidden

    @property
    def total_params(self):
        return self.layers * self.layer_params + 2 * self.vocab * self.hidden + self.hidden

    def layer_flops(self, tokens):
        """forward FLOPs of one layer for `tokens` tokens of sequences of length seq (causal attention counted at half)."""
        active_ffn = (3 if self.gated_ffn else 2) * self.hidden * self.ffn * (self.moe_topk if self.moe_experts else 1)
        return 2.0 * tokens * (self.attn_params + active_ffn) + 2.0 * tokens * self.seq * self.hidden


# ------------------------------------------------------------------------------------------------ memory + time models
def estimate_memory_gb(m, c, optimizer_bytes=6.0, hbm_reserve_gb=4.0):
    """Peak bytes per GPU for candidate `c` (dict).  Weights bf16 + grads bf16 (4 B / parameter) stay whole on the mp x pp shard unless
    sharding stage >= 2 / 3 splits them; the optimizer state (`optimizer_bytes` per parameter: int16 master residual + bf16 moments = 6 with
    split master weights, fp32 master + bf16 moments = 8, fp32 master + fp32 moments = 12) is divided by the sharding degree from stage 1 on."""
    mp, pp, sh, stage = c["mp"], c["pp"], c["sharding"], c.get("sharding_stage", 1)
    p_local = (m.total_params - 2 * m.vocab * m.hidden) / (mp * pp) + 2 * m.vocab * m.hidden / mp / (pp if pp > 1 else 1) * (2 if pp == 1 else 1)
    w = 2.0 * p_local / (sh if stage >= 3 else 1)
    g = 2.0 * p_local / (sh if stage >= 2 else 1)
    o = optimizer_bytes * p_local / (sh if sh > 1 else 1)
    mbs, seq, h = c["micro_batch"], m.seq, m.hidden
    sp = mp if c.get("sequence_parallel", mp > 1) else 1
    # saved activations of one layer with the lean fused blocks (kernels/fused_blocks.py): ~6.5 hidden-sized bf16 tensors per token at mp1
    # (~0.55 GB per 13B layer at micro-batch 2); 4 live on the residual stream (sharded by
    # sequence parallel), the rest are mp-sharded
    full_layer = mbs * seq * h * 2 * (4.0 / sp + 2.5 / mp)
    ckpt_layer = mbs * seq * h * 2 / sp
    rc = c.get("recompute", "none")
    per_layer = {"none": full_layer, "selective": ckpt_layer + 0.35 * (full_layer - ckpt_layer), "full": ckpt_layer}[rc]
    layers_local = m.layers / pp
    in_flight = 1
    if pp > 1:
        in_flight = {"FThenB": c["accumulate"], "1F1B": min(c["accumulate"], pp), "ZBH1": min(c["accumulate"], pp), "VPP": min(c["accumulate"], pp) * (1 + (pp - 1) / (pp * max(1, c.get("vpp", 1))))}[
            c.get("pp_schedule", "1F1B")]
    act = layers_local * per_layer * in_flight + (full_layer if rc == "full" else 0)
    logits = mbs * seq * m.vocab / mp * (2 + 4) if (pp == 1 or True) else 0
    return (w + g + o + act + logits) / GB + hbm_reserve_gb


def estimate_step_ms(m, c, cm=None, gemm_eff=0.68, attn_eff=0.18, global_batch=None):
    """Analytic step time of candidate `c`; the efficiencies are shares of the data-sheet bf16 rate that the own kernels reached on an
    H100 80GB HBM3 at 700 W (DESIGN.md §4): GEMMs of Llama-2-7B's 4096-row shapes 580 - 790 TFLOP/s (median ~680), causal attention
    forward + backward ~175 TFLOP/s."""
    cm = cm or CostModel()
    peak = cm.peaks.get("bf16_tflops_sustained", 989.0) * 1e9         # FLOP per ms
    mp, pp, sh, dp = c["mp"], c["pp"], c["sharding"], c["dp"]
    tok = c["micro_batch"] * m.seq
    dense = 2.0 * tok * (m.attn_params + (3 if m.gated_ffn else 2) * m.hidden * m.ffn * (m.moe_topk if m.moe_experts else 1)) / mp
    attn = 2.0 * tok * m.seq * m.hidden / mp
    fill = min(1.0, 0.80 + 0.20 * tok / 8192.0)                             # measured: 2048 / 4096 rows reach 0.84 / 0.88 of the 8192-row rate
    t_fwd = dense / (peak * gemm_eff * fill) + attn / (peak * attn_eff)
    rc = {"none": 0.0, "selective": 0.15, "full": 1.0}[c.get("recompute", "none")]
    t_layer = t_fwd * (3.0 + rc)
    if mp > 1:                                                            # 4 collectives per layer (fwd + bwd), mostly under the fused GEMMs
        exposed = 0.35 if c.get("sequence_parallel", True) else 1.0
        t_layer += 4 * cm.allreduce_ms(tok * m.hidden * 2, mp) * exposed
    layers_local = m.layers / pp
    t_mb = layers_local * t_layer + 3.0 * 2.0 * tok * m.vocab * m.hidden / mp / (peak * gemm_eff) / (pp if pp > 1 else 1)
    acc = c["accumulate"]
    bubble = 0.0
    if pp > 1:
        v = max(1, c.get("vpp", 1))
        bubble = {"FThenB": (pp - 1) / acc, "1F1B": (pp - 1) / acc, "VPP": (pp - 1) / (acc * v), "ZBH1": (pp - 1) / (3.0 * acc)}[c.get("pp_schedule", "1F1B")]
        t_mb += 2 * cm.mem_ms(tok * m.hidden * 2) * 4                       # activations / gradients over the hop
    p_local = m.total_params / (mp * pp)
    rep = dp * sh
    t_grad = cm.allreduce_ms(p_local * 2, rep) * (0.5 if c.get("sharding_stage", 1) >= 2 and sh > 1 else 1.0) * 0.5      # half hidden under backward
    t_opt = cm.mem_ms(p_local / (sh if sh > 1 else 1) * 16)
    t_gather = cm.allreduce_ms(p_local * 2, sh) * (0.5 if c.get("sharding_stage", 1) == 3 else 0.25) if sh > 1 else 0.0
    return acc * t_mb * (1.0 + bubble) + t_grad + t_opt + t_gather


# ------------------------------------------------------------------------------------------------ prune rules
_PRUNE_RULES = []
_HISTORY_RULES = []


def register_prune(fn):
    _PRUNE_RULES.append(fn)
    return fn


def register_history_prune(fn):
    _HISTORY_RULES.append(fn)
    return fn


@register_prune
def prune_by_degrees(t, c):
    return c["dp"] * c["mp"] * c["pp"] * c["sharding"] != t["num_gpus"]


@register_prune
def prune_by_mp(t, c):
    m = t["model"]
    if m.heads % c["mp"] or m.kv_heads % min(c["mp"], m.kv_heads) or m.vocab % c["mp"] or m.ffn % c["mp"]:
        return True
    return c["mp"] > t.get("gpus_per_node", 8)          # tensor parallel stays inside the NVSwitch domain


@register_prune
def prune_by_pp(t, c):
    m = t["model"]
    if m.layers % (c["pp"] * max(1, c.get("vpp", 1))):
        return True
    if c["pp"] == 1 and (c.get("vpp", 1) > 1 or c.get("pp_schedule", "1F1B") != "1F1B"):
        return True
    if c.get("pp_schedule") == "VPP" and c.get("vpp", 1) < 2:
        return True
    if c.get("pp_schedule") != "VPP" and c.get("vpp", 1) > 1:
        return True
    return c["pp"] > 1 and c["accumulate"] < c["pp"]      # fewer micro-batches than stages never fills the pipe


@register_prune
def prune_by_batch(t, c):
    rep = c["dp"] * c["sharding"]
    return t["global_batch"] % rep != 0 or (t["global_batch"] // rep) % c["micro_batch"] != 0


@register_prune
def prune_by_sharding(t, c):
    if c["sharding"] == 1 and c.get("sharding_stage", 1) != 1:
        return True
    return c.get("sharding_stage", 1) == 3 and c["pp"] > 1      # stage 3 re-gathers per layer: not combined with pipeline stages here


@register_prune
def prune_by_recompute(t, c):
    return c.get("sequence_parallel", False) and c["mp"] == 1


@register_prune
def prune_by_memory(t, c):
    c["mem_gb"] = round(estimate_memory_gb(t["model"], c, t.get("optimizer_bytes", 6.0)), 1)
    return c["mem_gb"] > t.get("hbm_gb", 80.0) * t.get("hbm_fraction", 0.94)


def _dominates(a, b):
    """True when candidate `a` needs at least as much memory as `b` in every respect (so an OOM of `b` implies an OOM of `a`)."""
    return (a["mp"] <= b["mp"] and a["pp"] <= b["pp"] and a["sharding"] <= b["sharding"] and a.get("sharding_stage", 1) <= b.get("sharding_stage", 1)
            and a["micro_batch"] >= b["micro_batch"] and {"none": 2, "selective": 1, "full": 0}[a.get("recompute", "none")] >= {"none": 2, "selective": 1, "full": 0}[b.get("recompute", "none")])


@register_history_prune
def prune_by_oom_history(t, c, history):
    return any(h.get("status") == "oom" and _dominates(c, h["cfg"]) for h in history)


@register_history_prune
def prune_by_seen(t, c, history):
    return any(_key(h["cfg"]) == _key(c) for h in history)


_KEYS = ("dp", "mp", "pp", "sharding", "sharding_stage", "micro_batch", "vpp", "recompute", "pp_schedule", "sequence_parallel")


def _key(c):
    return tuple(c.get(k) for k in _KEYS)


# ------------------------------------------------------------------------------------------------ search space
class SearchSpace:
    def __init__(self, tuner_cfg):
        t = dict(tuner_cfg)
        if "model" not in t:
            t["model"] = ModelSpec(t["hidden"], t["layers"], t["ffn"], t["vocab"], t["seq"], t.get("heads"), t.get("kv_heads"), t.get("gated_ffn", True),
                                   t.get("moe_experts", 0), t.get("moe_topk", 2))
        self.t = t

    def axis(self, name, default):
        v = self.t.get(name, "auto")
        if v == "auto" or v is None:
            return default
        return list(v) if isinstance(v, (list, tuple)) else [v]

    def candidates(self, history=()):
        t, n = self.t, self.t["num_gpus"]
        out, pruned = [], {}
        for mp, pp in itertools.product(self.axis("mp_degree", _divisors(n)), self.axis("pp_degree", _divisors(n))):
            if n % (mp * pp):
                continue
            rest = n // (mp * pp)
            for sh in self.axis("sharding_degree", _divisors(rest)):
                if rest % sh:
                    continue
                dp = rest // sh
                for stage, mbs, rc, sched, vpp in itertools.product(self.axis("sharding_stage", [1, 2, 3]), self.axis("micro_batch_size", [1, 2, 4, 8]),
                                                                   self.axis("recompute", ["none", "selective", "full"]),
                                                                   self.axis("pp_schedule", ["1F1B", "ZBH1", "VPP"]), self.axis("vpp_degree", [1, 2])):
                    rep = dp * sh
                    if t["global_batch"] % rep or (t["global_batch"] // rep) % mbs:
                        continue
                    c = dict(dp=dp, mp=mp, pp=pp, sharding=sh, sharding_stage=stage, micro_batch=mbs, accumulate=t["global_batch"] // rep // mbs, vpp=vpp, recompute=rc,
                             pp_schedule=sched, sequence_parallel=mp > 1)
                    reason = next((r.__name__ for r in _PRUNE_RULES if r(t, c)), None) or next((r.__name__ for r in _HISTORY_RULES if r(t, c, history)), None)
                    if reason:
                        pruned[reason] = pruned.get(reason, 0) + 1
                        continue
                    out.append(c)
        self.pruned = pruned
        return out


def rank(tuner_cfg, history=(), cm=None):
    """All surviving candidates with their memory and time estimates, fastest first."""
    space = SearchSpace(tuner_cfg)
    cm = cm or CostModel()
    cands = space.candidates(history)
    m = space.t["model"]
    for c in cands:
        c["est_ms"] = round(estimate_step_ms(m, c, cm), 2)
        c["est_tokens_per_s"] = round(space.t["global_batch"] * m.seq / c["est_ms"] * 1e3, 1)
    cands.sort(key=lambda c: c["est_ms"])
    return cands, space.pruned


def search(num_gpus, hidden, layers, ffn, vocab, seq, global_batch, heads=None, hbm_gb=80.0, bytes_per_param=12, measure=None, top_k=5, **extra):
    """Round-1 entry point: the `top_k` fastest candidates under the analytic model (or under `measure(cfg) -> ms`)."""
    cfg = dict(num_gpus=num_gpus, hidden=hidden, layers=layers, ffn=ffn, vocab=vocab, seq=seq, global_batch=global_batch, heads=heads, hbm_gb=hbm_gb,
               optimizer_bytes=bytes_per_param - 4, **extra)
    cands, _ = rank(cfg)
    if measure is not None:
        cands = cands[: max(top_k * 3, top_k)]
        for c in cands:
            c["measured_ms"] = measure(c)
        cands.sort(key=lambda c: c.get("measured_ms") or c["est_ms"])
    return cands[:top_k]


# ------------------------------------------------------------------------------------------------ history
class Recorder:
    """Trial history: one json line per trial, reloadable (resume), sorted views."""

    def __init__(self, path=None):
        self.path, self.history = path, []
        if path and os.path.exists(path):
            with open(path) as f:
                self.history = [json.loads(line) for line in f if line.strip()]

    def add(self, cfg, status="ok", metric=None, **info):
        rec = {"cfg": {k: v for k, v in cfg.items()}, "status": status, "metric": metric, "time": time.time(), **info}
        self.history.append(rec)
        if self.path:
            os.makedirs(os.path.dirname(os.path.abspath(self.path)), exist_ok=True)
            with open(self.path, "a") as f:
                f.write(json.dumps(rec) + "\n")
        return rec

    def sorted(self, higher_is_better=True):
        ok = [h for h in self.history if h["status"] == "ok" and h.get("metric") is not None]
        return sorted(ok, key=lambda h: h["metric"], reverse=higher_is_better)

    def best(self, higher_is_better=True):
        s = self.sorted(higher_is_better)
        return s[0] if s else None

    def to_csv(self, path):
        cols = list(_KEYS) + ["accumulate", "mem_gb", "est_ms", "status", "metric"]
        with open(path, "w") as f:
            f.write(",".join(cols) + "\n")
            for h in self.history:
                row = dict(h["cfg"], status=h["status"], metric=h.get("metric"))
                f.write(",".join("" if row.get(c) is None else str(row.get(c)) for c in cols) + "\n")


# ------------------------------------------------------------------------------------------------ driver
def cfg_to_env(c):
    """Environment a trial process reads (bench.py / a user script): the candidate in B200_TUNE_* variables + one JSON blob."""
    env = {f"B200_TUNE_{k.upper()}": str(v) for k, v in c.items() if k in _KEYS or k == "accumulate"}
    env["B200_TUNE_CFG"] = json.dumps({k: c[k] for k in c if k in _KEYS or k == "accumulate"})
    return env


class AutoTuner:
    """search_once() hands out the best not-yet-tried candidate (history-pruned); add_cfg() / record() feed results back; tune() runs the loop."""

    def __init__(self, tuner_cfg, history_path=None):
        self.cfg = dict(tuner_cfg)
        self.recorder = Recorder(history_path if history_path is not None else self.cfg.get("history_path"))
        self.history = self.recorder.history         # resumed trials prune and are never repeated
        self._cm = CostModel()
        self._pending = []

    def search_once(self):
        """The best candidate that has neither been tried nor handed out before (None when the space is exhausted)."""
        pending = [{"cfg": c, "status": "pending"} for c in self._pending]
        cands, self.pruned = rank(self.cfg, list(self.history) + pending, self._cm)
        if not cands:
            return None
        self._pending.append(cands[0])
        return cands[0]

    def add_cfg(self, cfg, status="ok", metric=None, **info):
        self._pending = [c for c in self._pending if _key(c) != _key(cfg)]
        return self.recorder.add(cfg, status, metric, **info)

    record = add_cfg

    def best(self):
        return self.recorder.best(self.cfg.get("higher_is_better", True))

    def tune(self, run=None, command=None, max_trials=8, max_time_s=None, timeout_s=1800, metric_key="value"):
        """Trial loop.  `run(cfg) -> metric | ("oom", None) | raises`, or `command` (list / str): a subprocess per candidate that prints one
        JSON line containing `metric_key` (bench.py's line works); an out-of-memory message in its output marks the trial "oom"."""
        t0 = time.time()
        for _ in range(max_trials):
            if max_time_s is not None and time.time() - t0 > max_time_s:
                break
            c = self.search_once()
            if c is None:
                break
            try:
                if run is not None:
                    res = run(c)
                    status, metric = ("oom", None) if res == "oom" or (isinstance(res, tuple) and res[0] == "oom") else ("ok", float(res))
                else:
                    status, metric = self._run_command(c, command, timeout_s, metric_key)
            except MemoryError:
                status, metric = "oom", None
            except Exception as e:  # noqa: BLE001
                status, metric = "error", None
                self.add_cfg(c, status, metric, error=str(e)[:300])
                continue
            self.add_cfg(c, status, metric)
        return self.best()

    @staticmethod
    def _run_command(c, command, timeout_s, metric_key):
        env = dict(os.environ, **cfg_to_env(c))
        try:
            r = subprocess.run(command, shell=isinstance(command, str), capture_output=True, text=True, env=env, timeout=timeout_s)
        except subprocess.TimeoutExpired:
            return "timeout", None
        text = r.stdout + r.stderr
        if "out of memory" in text.lower() or "CUDA_ERROR_OUT_OF_MEMORY" in text:
            return "oom", None
        for line in reversed(r.stdout.splitlines()):
            line = line.strip()
            if line.startswith("{") and metric_key in line:
                try:
                    return "ok", float(json.loads(line)[metric_key])
                except Exception:  # noqa: BLE001
                    continue
        return ("error" if r.returncode else "no_metric"), None
