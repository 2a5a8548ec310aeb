"""bench.py --dump-outputs: names, dtypes, total size <= 64 MB, identical arrays from two identical runs."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = {"pred", "features", "loss", "params_sample", "grads_sample", "sample_index"}


def _run(out_dir, steps):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps),
                        "--warmup", "3", "--batch", "32", "--num-batches", "2", "--no-cpu-baseline",
                        "--dump-outputs", str(out_dir)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1
    return json.loads(lines[0])


def test_dump_outputs_names_dtypes_size_and_repeatability(tmp_path):
    a, b = tmp_path / "a", tmp_path / "b"
    da, db = _run(a, 3), _run(b, 3)
    assert da["steps"] == db["steps"] == 3
    files = sorted(os.listdir(a))
    assert {f[:-4] for f in files} == NAMES and all(f.endswith(".npy") for f in files)
    assert sum(os.path.getsize(a / f) for f in files) <= 64 << 20
    for f in files:
        x, y = np.load(a / f), np.load(b / f)
        assert x.dtype in (np.float32, np.float64), (f, x.dtype)
        assert np.isfinite(x).all(), f
        np.testing.assert_array_equal(x, y, err_msg=f)
    assert np.load(a / "pred.npy").shape == (32, 1) and np.load(a / "features.npy").shape == (32, 2048)
