"""distributed.auto_tuner: search space, prune rules (static + history based), memory / time models, recorder, trial loop.
Parity model: test/auto_parallel/test_auto_tuner*.py (prune / search / recorder unit tests)."""
import json
import sys

import pytest

from paddle_b200.distributed import auto_tuner as AT

LLAMA13B = dict(num_gpus=8, hidden=5120, layers=40, ffn=13824, vocab=32000, seq=4096, global_batch=32, heads=40, optimizer_bytes=6.0)


def test_model_spec_counts_llama_13b():
    m = AT.ModelSpec(5120, 40, 13824, 32000, 4096, heads=40)
    assert abs(m.total_params - 13.0e9) / 13.0e9 < 0.01
    assert m.layer_flops(4096) > 2 * 4096 * m.layer_params * 0.99


def test_memory_model_matches_the_measured_single_gpu_footprint():
    m = AT.ModelSpec(5120, 40, 13824, 32000, 4096, heads=40)
    c = dict(dp=1, mp=1, pp=1, sharding=1, sharding_stage=1, micro_batch=2, accumulate=2, recompute="none", pp_schedule="1F1B", vpp=1, sequence_parallel=False)
    gb = AT.estimate_memory_gb(m, c, optimizer_bytes=6.0)
    assert 150 < gb < 166, gb                                    # 130 GB of state + activations: far beyond one 80 GB GPU
    c12 = dict(c)
    assert AT.estimate_memory_gb(m, c12, optimizer_bytes=12.0) > 180          # classic fp32 master + fp32 moments does not fit one GPU
    assert AT.estimate_memory_gb(m, dict(c, recompute="full")) < gb
    assert AT.estimate_memory_gb(m, dict(c, mp=2, sequence_parallel=True)) < 0.62 * gb


def test_prune_rules_by_name():
    t = dict(LLAMA13B, model=AT.ModelSpec(5120, 40, 13824, 32000, 4096, heads=40))
    ok = dict(dp=2, mp=2, pp=2, sharding=1, sharding_stage=1, micro_batch=2, accumulate=8, vpp=1, recompute="none", pp_schedule="ZBH1", sequence_parallel=True)
    assert not any(r(t, dict(ok)) for r in AT._PRUNE_RULES)
    assert AT.prune_by_degrees(t, dict(ok, dp=4))
    assert AT.prune_by_mp(t, dict(ok, mp=3)) and AT.prune_by_mp(t, dict(ok, mp=16))
    assert AT.prune_by_pp(t, dict(ok, pp=3)) and AT.prune_by_pp(t, dict(ok, pp_schedule="VPP", vpp=1)) and AT.prune_by_pp(t, dict(ok, accumulate=1))
    assert AT.prune_by_pp(t, dict(ok, pp=1, pp_schedule="ZBH1"))
    assert AT.prune_by_batch(t, dict(ok, micro_batch=3))
    assert AT.prune_by_sharding(t, dict(ok, sharding_stage=2)) and AT.prune_by_sharding(t, dict(ok, sharding=2, dp=1, sharding_stage=3))
    big = dict(ok, dp=8, mp=1, pp=1, pp_schedule="1F1B", accumulate=2, sequence_parallel=False, micro_batch=8)
    assert AT.prune_by_memory(t, big) and big["mem_gb"] > 180


def test_rank_prefers_sensible_layouts_and_reports_pruning():
    cands, pruned = AT.rank(LLAMA13B)
    assert cands and pruned.get("prune_by_memory", 0) > 0 and pruned.get("prune_by_pp", 0) > 0
    assert all(c["dp"] * c["mp"] * c["pp"] * c["sharding"] == 8 and c["mem_gb"] <= 80 * 0.94 for c in cands)
    assert cands[0]["est_ms"] <= cands[-1]["est_ms"]
    best = cands[0]
    assert best["mp"] <= 4 and best["recompute"] != "full"                       # no needless recompute / tensor parallel at 8 GPUs with 80 GB
    same = [c for c in cands if (c["dp"], c["mp"], c["pp"], c["sharding"], c["micro_batch"], c["recompute"]) == (2, 2, 2, 1, 2, "none")]
    by = {c["pp_schedule"]: c["est_ms"] for c in same if c["vpp"] in (1, 2)}
    assert by["ZBH1"] < by["1F1B"]                                                # zero-bubble beats 1F1B at equal layout
    res = AT.search(**{k: v for k, v in LLAMA13B.items() if k != "optimizer_bytes"}, bytes_per_param=12, top_k=3)
    assert len(res) == 3 and res[0]["est_ms"] <= res[2]["est_ms"]


def test_history_prunes_dominated_and_seen_configs(tmp_path):
    path = str(tmp_path / "hist.jsonl")
    t = AT.AutoTuner(dict(LLAMA13B, history_path=path))
    first = t.search_once()
    t.add_cfg(first, "oom")
    second = t.search_once()
    assert second is not None and AT._key(second) != AT._key(first) and not AT._dominates(second, first)
    assert t.pruned.get("prune_by_oom_history", 0) >= 1
    t.add_cfg(second, "ok", metric=80000.0)
    t2 = AT.AutoTuner(dict(LLAMA13B), history_path=path)                            # resume: nothing is tried twice
    third = t2.search_once()
    assert AT._key(third) not in (AT._key(first), AT._key(second)) and len(t2.history) == 2
    assert t2.best()["metric"] == 80000.0
    t2.recorder.to_csv(str(tmp_path / "h.csv"))
    rows = open(tmp_path / "h.csv").read().strip().splitlines()
    assert rows[0].startswith("dp,mp,pp") and len(rows) == 3 and ",oom," in rows[1]


def test_tune_loop_with_callable_and_with_a_command(tmp_path):
    calls = []

    def run(cfg):
        calls.append(cfg)
        if cfg["micro_batch"] >= 4:
            return "oom"
        return 1e6 / cfg["est_ms"]

    t = AT.AutoTuner(dict(LLAMA13B))
    best = t.tune(run=run, max_trials=5)
    assert len(calls) == 5 and best is not None and best["status"] == "ok"
    assert best["metric"] == max(h["metric"] for h in t.history if h["status"] == "ok")
    script = tmp_path / "trial.py"
    script.write_text("import os, json\n"
                      "c = json.loads(os.environ['B200_TUNE_CFG'])\n"
                      "assert os.environ['B200_TUNE_MP'] == str(c['mp'])\n"
                      "if c['pp'] > 1: print('RuntimeError: CUDA out of memory'); raise SystemExit(1)\n"
                      "print(json.dumps({'value': 1000.0 * c['mp'], 'unit': 'tokens/s'}))\n")
    t = AT.AutoTuner(dict(LLAMA13B, pp_degree=[1, 2], mp_degree=[2, 4], micro_batch_size=[1], recompute=["none"], sharding_stage=[1], pp_schedule=["1F1B"], vpp_degree=[1]))
    best = t.tune(command=[sys.executable, str(script)], max_trials=6, timeout_s=60)
    st = {h["status"] for h in t.history}
    assert "ok" in st and best["cfg"]["pp"] == 1 and best["metric"] == 1000.0 * best["cfg"]["mp"]
    assert all(h["cfg"]["pp"] == 1 for h in t.history if h["status"] == "ok")
    env = AT.cfg_to_env(best["cfg"])
    assert json.loads(env["B200_TUNE_CFG"])["mp"] == best["cfg"]["mp"]


def test_launch_auto_tuner_mode(tmp_path):
    """`python -m paddle_b200.distributed.launch --auto_tuner_json`: every trial is a real launch of the script (1 process here); the script reads the
    candidate from the environment and prints its metric; the history lands in the log dir."""
    import os
    import subprocess

    script = tmp_path / "train.py"
    script.write_text("import os, json\n"
                      "c = json.loads(os.environ['B200_TUNE_CFG'])\n"
                      "assert os.environ.get('PADDLE_TRAINER_ID') is not None\n"
                      "print(json.dumps({'value': 100.0 + 10 * c['micro_batch'] - (50 if c['recompute'] == 'full' else 0)}))\n")
    cfg = dict(num_gpus=1, hidden=1024, layers=8, ffn=4096, vocab=32000, seq=2048, global_batch=8, heads=8, micro_batch_size=[1, 2], recompute=["none", "full"],
               max_trials=4, trial_timeout_s=120)
    (tmp_path / "tuner.json").write_text(json.dumps(cfg))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "paddle_b200.distributed.launch", "--nproc_per_node", "1", "--log_dir", str(tmp_path / "log"), "--auto_tuner_json",
                        str(tmp_path / "tuner.json"), str(script)], capture_output=True, text=True, cwd=root, timeout=600, env=dict(os.environ, PYTHONPATH=root))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out = json.loads([line for line in r.stdout.splitlines() if line.startswith('{"auto_tuner_best"')][-1])
    assert out["trials"] == 4 and out["auto_tuner_best"]["metric"] == 120.0 and out["auto_tuner_best"]["cfg"]["micro_batch"] == 2
    hist = [json.loads(line) for line in open(tmp_path / "log" / "auto_tuner_history.jsonl")]
    assert len(hist) == 4 and all(h["status"] == "ok" for h in hist)
    assert os.path.exists(tmp_path / "log" / "auto_tuner_history.csv")
