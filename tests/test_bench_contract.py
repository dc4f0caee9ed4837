"""bench.py's output contract (no GPU): the reference arm really runs here on the CPU (one bounded step) and prints ONE JSON
line with the agreed keys; the committed bench lines under profiles/ carry every key a reader of them needs."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE_KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
             "dtype", "data", "config", "e2e", "cpu_baseline"}


def test_reference_arm_prints_one_contract_line():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    d = json.loads(lines[0])
    assert BASE_KEYS <= set(d) and d["impl"] == "reference"
    assert d["metric"] == "LR event-frames/sec" and d["unit"] == "frames/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["e2e"]["value"] == d["value"]
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["cpu_baseline"]["kind"] in ("port", "reference") and d["cpu_baseline"]["cores"] >= 1
    assert "workload" in d["config"]


def test_committed_bench_lines_have_every_key():
    for name in ("bench_cfg2_n1.json",):
        d = json.load(open(os.path.join(ROOT, "profiles", name)))
        assert (BASE_KEYS - {"cpu_baseline"}) <= set(d), name
        assert {"clocks", "gpu_launches", "roofline"} <= set(d), name
        assert {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"} <= set(d["e2e"]), name
        assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] != d["value"], name
        assert {"bound", "achieved", "peak", "unit", "frac", "traffic"} <= set(d["roofline"]), name
        assert abs(d["roofline"]["frac"] - d["roofline"]["achieved"] / d["roofline"]["peak"]) < 1e-9, name
        assert {"sm_mhz", "sm_max_mhz", "reasons"} <= set(d["clocks"]) and not set(d["clocks"]["reasons"]) & {
            "hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown"}, name
        assert d["gpu_launches"] > 0 and d["config"]["workload"], name
    d = json.load(open(os.path.join(ROOT, "profiles", "bench_cfg2_n1.json")))
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d["cpu_baseline"])


def test_round2_bench_lines_carry_parity_rooflines_and_every_config():
    """The committed line: the parity check of the measured plan, the family (not best-launch) roofline with the best launch kept
    beside it, the HBM rooflines of the byte-bound stages, cfg3 / cfg4 with their own parity and CPU baseline, the cfg5 sweep with
    a CPU column, and the reference arm's line for the same workload."""
    for name in ("bench_cfg2_n1.json",):
        d = json.load(open(os.path.join(ROOT, "profiles", name)))
        assert (BASE_KEYS - {"cpu_baseline"}) <= set(d) and {"clocks", "gpu_launches", "roofline", "parity", "roofline_hbm", "configs"} <= set(d), name
        assert d["parity"]["ok"] and d["parity"]["rel_max"] <= 1e-3 and d["parity"]["windows"] == 6, name
        r = d["roofline"]
        assert {"bound", "achieved", "peak", "unit", "frac", "traffic", "largest_launch", "best_launch", "per_layer"} <= set(r), name
        assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9 and r["frac"] < r["best_launch"]["frac"], name
        assert {"scatter", "redistribute", "small_convs", "elementwise"} <= set(d["roofline_hbm"]), name
        for cfg, windows in (("cfg3", 6), ("cfg4", 14)):
            c = d["configs"][cfg]
            assert c["parity"]["ok"] and c["parity"]["windows"] == windows and c["value"] > 0 and c["e2e"]["value"] > 0, (name, cfg)
        assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0 and d["e2e"]["value"] != d["value"], name
    d1 = json.load(open(os.path.join(ROOT, "profiles", "bench_cfg2_n1.json")))
    assert {"value", "unit", "cores", "kind", "sample"} <= set(d1["cpu_baseline"])
    assert all("cpu_baseline" in d1["configs"][c] for c in ("cfg3", "cfg4"))
    ops = {(p["op"], p["events"] >= 5_000_000) for p in d1["sweep"]}
    assert ("scatter_cnt", True) in ops and ("cnt2event", True) in ops and any("cpu_Mev_per_s" in p for p in d1["sweep"])
    ref = json.load(open(os.path.join(ROOT, "profiles", "bench_cfg2_reference.json")))
    assert ref["impl"] == "reference" and ref["metric"] == d1["metric"] and ref["config"]["workload"] == d1["config"]["workload"]


@pytest.mark.skipif(not os.path.exists(os.path.join(ROOT, "profiles", "bench_cfg2_n2.json")),
                    reason="needs a bench line recorded on two GPUs (profiles/bench_cfg2_n2.json)")
def test_two_gpu_bench_line_scales_and_checks_the_exchange():
    """At N = 2: weak scaling of the inference value, and the training iteration captured with its NCCL exchange plus the
    hardware check of the result."""
    d1 = json.load(open(os.path.join(ROOT, "profiles", "bench_cfg2_n1.json")))
    d2 = json.load(open(os.path.join(ROOT, "profiles", "bench_cfg2_n2.json")))
    assert d2["n_gpus"] == 2 and 1.9 < d2["value"] / d1["value"] < 2.1
    for t in (d2["train"], d2["configs"]["cfg3"]["train"], d2["configs"]["cfg4"]["train"]):
        assert "NCCL" in t["mode"] and t["gradient_exchange_check"]["ok"] and t["gradient_exchange_check"]["identical_on_all_ranks"]


def test_dump_outputs_writes_seeded_samples_within_the_budget(tmp_path):
    """--dump-outputs: every array lands as <name>.npy in float32, the total stays within the budget, and an array that does not
    fit is reduced to the same seeded row sample (with its row indices) on every call, so two runs compare output for output."""
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    import bench
    budget = 1 << 20
    arrays = {"sr_counts": torch.arange(2 * 2 * 64 * 64, dtype=torch.float32).view(2, 2, 64, 64),
              "events": torch.arange(100000 * 4, dtype=torch.float64).view(1, 100000, 4)}
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), arrays, budget=budget)
    files = sorted(p.name for p in (tmp_path / "a").iterdir())
    assert files == ["events.npy", "events_rows.npy", "sr_counts.npy"]
    assert sum(p.stat().st_size for p in (tmp_path / "a").iterdir()) <= budget + 3 * 128      # + the three .npy headers
    sr = np.load(tmp_path / "a" / "sr_counts.npy")
    assert sr.dtype == np.float32 and np.array_equal(sr, arrays["sr_counts"].numpy())
    ev, rows = np.load(tmp_path / "a" / "events.npy"), np.load(tmp_path / "a" / "events_rows.npy")
    assert ev.dtype == np.float32 and rows.dtype == np.float64 and 0 < len(rows) < 100000 and np.all(np.diff(rows) > 0)
    assert np.array_equal(ev, arrays["events"].view(-1, 4).numpy()[rows.astype(np.int64)].astype(np.float32))
    for n in files:
        assert np.array_equal(np.load(tmp_path / "a" / n), np.load(tmp_path / "b" / n)), n


def test_dump_outputs_is_refused_for_the_reference_arm(tmp_path):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--dump-outputs", str(tmp_path)],
                       capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode != 0 and "--dump-outputs" in r.stderr and not any(tmp_path.iterdir())
