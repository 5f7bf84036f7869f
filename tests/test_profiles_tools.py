"""The committed evidence under profiles/ stays machine-readable: the bench lines parse and carry the contract keys, and
the generator that turns them into the results table runs on them (CPU only, no GPU, no reference)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROF = os.path.join(ROOT, "profiles")
CONTRACT = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
            "dtype", "data", "config", "e2e", "gpu_launches", "clocks", "roofline", "cpu_baseline"]


def _line(name):
    with open(os.path.join(PROF, name)) as fh:
        rows = [ln for ln in fh.read().splitlines() if ln.startswith("{")]
    assert len(rows) == 1, "%s: expected exactly one JSON line" % name
    return json.loads(rows[0])


def test_committed_bench_lines_follow_the_contract():
    for cfg in ("second", "pillars", "cbgs"):
        d = _line("h100_bench_%s.json" % cfg)
        assert [k for k in CONTRACT if k not in d] == []
        assert d["config"]["baseline_config"] == cfg and d["n_gpus"] == 1 and d["data"] == "synthetic"
        r = d["roofline"]
        assert r["bound"] == "tensor" and abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-9
        e = d["e2e"]
        assert e["h2d_bytes_per_step"] > 0 and e["d2h_bytes_per_step"] > 0 and e["value"] < d["value"]
        assert d["cpu_baseline"]["kind"] in ("port", "reference") and d["cpu_baseline"]["cores"] >= 1
        g = d["stage_ms_per_step_in_graph"]
        assert g and abs(sum(g.values()) - d["ms_per_step"]) < 0.05 * d["ms_per_step"]      # the stages add up to the step
    out = subprocess.run([sys.executable, os.path.join(PROF, "make_results.py")] +
                         [os.path.join(PROF, "h100_bench_%s.json" % c) for c in ("second", "pillars", "cbgs")],
                         capture_output=True, text=True, check=True).stdout
    assert "| second |" in out and "inside the replayed CUDA graph" in out
