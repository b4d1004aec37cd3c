"""bench.py --dump-outputs: the last timed step's outputs, float32, within the 64 MB limit, identical between two runs with
the same arguments (seeded inputs, parameters and dropout masks)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
ROOT = Path(__file__).resolve().parents[1]
DIMS = [128, 256, 256, 40]


def _run(out):
    p = subprocess.run([sys.executable, str(ROOT / "bench.py"), "--gpus", "1", "--steps", "2", "--warmup", "1", "--no-parity",
                        "--no-cpu-baseline", "--dump-outputs", str(out)], capture_output=True, text=True, timeout=800,
                       cwd=str(ROOT))
    assert p.returncode == 0, p.stderr[-3000:]
    return {f.stem: np.load(f) for f in sorted(Path(out).glob("*.npy"))}


def test_dump_outputs_file_set_dtype_size_and_repeatability(tmp_path):
    a, b = _run(tmp_path / "a"), _run(tmp_path / "b")
    params = {f"param.convs.{l}.{k}" for l in range(3) for k in ("weight", "bias")}
    params |= {f"param.bns.{l}.{k}" for l in range(2) for k in ("weight", "bias", "running_mean", "running_var")}
    assert set(a) == {"loss", "logits", "grads"} | params
    assert all(v.dtype == np.float32 for v in a.values())
    assert sum(v.nbytes for v in a.values()) <= 64 << 20
    n_par = sum(DIMS[l] * DIMS[l + 1] + DIMS[l + 1] for l in range(3)) + sum(2 * DIMS[l + 1] for l in range(2))
    assert a["loss"].shape == (3,) and a["grads"].shape == (n_par,) and a["logits"].shape[1] == 40
    assert a["param.convs.0.weight"].shape == (128, 256)
    assert np.isfinite(a["loss"]).all() and np.isfinite(a["logits"]).all()
    for k in a:
        assert np.array_equal(a[k], b[k]), k
