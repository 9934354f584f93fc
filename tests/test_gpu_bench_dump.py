"""bench.py --dump-outputs: the planes of the last timed step, written as float64 .npy files, are the same from run to
run on the same arguments, agree with the JSON line, and stay within the size budget."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.normpath(os.path.join(os.path.dirname(__file__), ".."))


def _run(out_dir, steps):
    cmd = [sys.executable, os.path.join(ROOT, "bench.py"), "--workload", "c2", "--scale", "0.01", "--steps", str(steps), "--warmup", "1",
           "--no-e2e", "--no-cpu-baseline", "--no-extras", "--dump-outputs", str(out_dir)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-3000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, lines
    return json.loads(lines[0])


def test_dump_outputs_repeatable_and_bounded(tmp_path):
    a, b = tmp_path / "a", tmp_path / "b"
    la, lb = _run(a, 2), _run(b, 3)
    assert la["steps"] == 2 and lb["steps"] == 3
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b)) and "cell_val.npy" in names and "rec_commit_lsn.npy" in names
    assert sum(os.path.getsize(a / n) for n in names) <= 64 << 20
    for n in names:
        x, y = np.load(a / n), np.load(b / n)
        assert x.dtype in (np.float32, np.float64) and np.array_equal(x, y), n
    summ = np.load(a / "summary.npy")
    n_records = int(summ[0, 0]) * 2**32 + int(summ[0, 1])
    assert n_records == la["config"]["records"] > 0
