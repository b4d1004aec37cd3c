"""bench.py's output contract, checked on the CPU-only arm (`--impl reference`): exactly one line on stdout, valid JSON,
the keys a consumer reads.  (The GPU arm prints the same keys plus roofline / clocks; it is exercised on the GPU.)"""
import json
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parents[1]


@pytest.mark.timeout(600)
def test_reference_arm_prints_exactly_one_json_line():
    p = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=580, cwd=str(ROOT))
    assert p.returncode == 0, p.stderr[-2000:]
    lines = [l for l in p.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, p.stdout[:500]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "edges/s" and d["higher_is_better"] is True
    assert d["n_gpus"] == 1 and d["steps"] == 1 and d["value"] > 0 and d["ms_per_step"] > 0
    assert "ARXIV-shape" in d["metric"] and d["config"]["workload"].startswith("configs[1]")
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and cb["scatter_add_value"] > 0
    assert d["e2e"] == {"value": d["value"], "unit": "edges/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["gpu_launches"] == 0 and d["vs_baseline"] is None and d["scaling"] == "strong"
    assert set(d["config"]) == {"workload", "edges_per_step", "nnz_walked", "l2_policy"}       # the same keys as the GPU arm


def test_reference_arm_is_silent_on_non_zero_ranks():
    import os
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    p = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "1"],
                       capture_output=True, text=True, timeout=120, cwd=str(ROOT), env=env)
    assert p.returncode == 0 and p.stdout.strip() == ""


def test_dump_outputs_is_rejected_for_the_reference_arm(tmp_path):
    p = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                        "--dump-outputs", str(tmp_path / "d")], capture_output=True, text=True, timeout=120, cwd=str(ROOT))
    assert p.returncode == 2 and p.stdout.strip() == "", p.stderr[-2000:]
    assert "--dump-outputs" in p.stderr and not (tmp_path / "d").exists()
