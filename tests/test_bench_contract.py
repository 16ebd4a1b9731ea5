"""bench.py on the smallest workload: the JSON line of the reference arm carries the contract keys (CPU tier); the
GPU arm's --dump-outputs files (GPU tier)."""
import json
import os
import subprocess
import sys

import pytest

from helpers import ROOT


def test_reference_arm_json_contract():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "mini",
                        "--steps", "1", "--warmup", "0", "--cpu-seconds", "1"], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [l for l in r.stdout.splitlines() if l.strip()]
    assert len(lines) == 1, r.stdout                                  # exactly one JSON line on stdout
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
              "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert k in d, k
    assert d["impl"] == "reference" and d["unit"] == "steps/s" and d["higher_is_better"] is True
    assert d["vs_baseline"] is None and d["dtype"] == "f32" and d["data"] == "synthetic"
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1 and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": "steps/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert d["value"] > 0 and "workload" in d["config"]


@pytest.mark.gpu
def test_dump_outputs_are_small_float_arrays_identical_across_runs(tmp_path):
    """--dump-outputs: after the timed steps, the outputs of the last one as float32 / float64 .npy files, at most 64 MB
    in all, bit-identical between two runs with the same arguments; --steps sets the number of timed steps."""
    import numpy as np
    steps = 7
    dumps = []
    for k in range(2):
        out = tmp_path / f"d{k}"
        r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--workload", "mini", "--steps", str(steps),
                            "--warmup", "2", "--extra-modes", "", "--no-dense-extra", "--no-cpu-baseline",
                            "--dump-outputs", str(out)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        line = [l for l in r.stdout.splitlines() if l.strip()]
        assert len(line) == 1 and json.loads(line[0])["steps"] == steps
        files = sorted(os.listdir(out))
        assert files and all(f.endswith(".npy") for f in files)
        assert sum(os.path.getsize(out / f) for f in files) <= 64 << 20
        arrs = {f: np.load(out / f) for f in files}
        assert all(a.dtype in (np.float32, np.float64) for a in arrs.values())
        assert len(arrs["picks.npy"]) == steps
        dumps.append(arrs)
    assert dumps[0].keys() == dumps[1].keys()
    for f in dumps[0]:
        assert np.array_equal(dumps[0][f], dumps[1][f]), f
