"""CPU tests of ModelPicker's epsilon search (coda_b200.eps_search): the realisations, the metrics and selection against
the reference script's own code (tests/golden/eps_search_*.npz, made by tests/golden/make_eps_search_golden.py), the
command line with a scripted search, the CODA_B200_TASK_EPS hook of main.py's dispatch, and the new C ABI."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN, ROOT


def test_realisations_are_the_scripts_numpy_draws():
    from coda_b200.eps_search import create_realisations
    np.random.seed(17)
    got = create_realisations(300, 7, 40)
    np.random.seed(17)
    want = np.array([np.random.permutation(300)[:40] for _ in range(7)])
    assert np.array_equal(got, want) and got.shape == (7, 40)
    assert all(len(set(row)) == 40 for row in got.tolist())


@pytest.mark.parametrize("case", ["crafted", "random"])
def test_metrics_and_selection_match_the_reference_script(case):
    from coda_b200.eps_search import search_metrics
    g = np.load(os.path.join(GOLDEN, f"eps_search_{case}.npz"))
    eps = g["epsilons"].tolist()
    best_avg, best_fast, metrics = search_metrics(g["best"], g["pool_acc"], int(g["pool_size"]), eps,
                                                  float(g["threshold"]))
    assert list(metrics) == eps
    for e, x in enumerate(eps):
        m = metrics[x]
        assert m["success_mean"] == g["success_mean"][e].tolist(), (case, x)
        assert m["acc_mean"] == g["acc_mean"][e].tolist(), (case, x)
        assert m["avg_success"] == float(g["avg_success"][e])
        assert float(m["fastest_t"]) == float(g["fastest_t"][e])
    assert (best_avg, best_fast) == (float(g["best_avg"]), float(g["best_fast"]))
    if case == "crafted":                                 # the cases the fixture was made to hold
        ft = g["fastest_t"]
        assert ft[0] == ft[1] == 0 and np.isinf(ft[2]) and np.isinf(ft[3])
        assert g["success_mean"][3].max() >= float(g["threshold"])          # reached, but not when smoothed
        assert best_avg == best_fast == eps[0]                              # the first of two tied epsilons


def test_run_keys_are_stable_and_distinct():
    from coda_b200.eps_search import eps_search_run_key
    keys = {eps_search_run_key(5, e, r) for e in range(15) for r in range(300)}
    assert len(keys) == 15 * 300 and all(0 <= k < 1 << 64 for k in keys)
    assert eps_search_run_key(5, 3, 7) == eps_search_run_key(5, 3, 7) != eps_search_run_key(6, 3, 7)
    assert eps_search_run_key(-1, 0, 0) == eps_search_run_key((1 << 64) - 1, 0, 0)


def _fake_search(calls):
    def search(dataset, epsilons, iterations, pool_size, budget, threshold, seed):
        calls.append(dict(shape=tuple(dataset.preds.shape), epsilons=epsilons, iterations=iterations,
                          pool_size=pool_size, budget=budget, threshold=threshold, seed=seed,
                          np_draw=float(np.random.random())))
        metrics = {e: {"success_mean": [0.5], "acc_mean": [0.7], "avg_success": 0.5, "fastest_t": float("inf")}
                   for e in epsilons}
        return {"best_avg": epsilons[-1], "best_fast": epsilons[0], "metrics": metrics}
    return search


def test_cli_writes_and_skips_best_epsilons(tmp_path, monkeypatch):
    from coda_b200.eps_search import main
    from coda_b200.synth import synth
    d = tmp_path / "data"
    d.mkdir()
    for name, seed in (("taskA", 1), ("taskB", 2)):
        preds, labels = synth(4, 30, 3, seed=seed)
        torch.save(preds, d / f"{name}.pt")
        torch.save(labels, d / f"{name}_labels.pt")
    monkeypatch.chdir(tmp_path)
    calls = []
    assert main(["--task", "taskA", "--pred-dir", str(d), "--epsilons", "0.4,0.45", "--iterations", "3",
                 "--pool-size", "20", "--budget", "10", "--threshold", "0.8", "--seed", "4"],
                search=_fake_search(calls)) == 0
    np.random.seed(4)
    assert calls == [dict(shape=(4, 30, 3), epsilons=[0.4, 0.45], iterations=3, pool_size=20, budget=10,
                          threshold=0.8, seed=4, np_draw=float(np.random.random()))]
    out = json.loads((tmp_path / "best_epsilons.json").read_text())
    assert out == {"taskA": {"best_avg": 0.45, "best_fast": 0.4}}
    # a key already there is skipped; the directory mode keys by file name and ignores *_labels.pt
    assert main(["--task", "taskA", "--pred-dir", str(d)], search=_fake_search(calls)) == 0
    assert len(calls) == 1
    assert main(["--pred-dir", str(d), "--epsilons", "0.3"], search=_fake_search(calls)) == 0
    out = json.loads((tmp_path / "best_epsilons.json").read_text())
    assert out == {"taskA": {"best_avg": 0.45, "best_fast": 0.4}, "taskA.pt": {"best_avg": 0.3, "best_fast": 0.3},
                   "taskB.pt": {"best_avg": 0.3, "best_fast": 0.3}}
    assert [c["shape"] for c in calls] == [(4, 30, 3)] * 3
    assert calls[1]["epsilons"] == [0.3] and calls[1]["iterations"] == 1000 and calls[1]["seed"] is None
    with pytest.raises(ValueError):
        main(["--task", "taskB", "--pred-dir", str(d), "--epsilons", "0.4,1.0"], search=_fake_search(calls))
    assert len(calls) == 3


def test_the_search_refuses_without_a_gpu_slab():
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200 import TensorDataset
    from coda_b200.synth import synth
    preds, _ = synth(4, 30, 3, seed=1)
    with pytest.raises(ValueError):
        modelpicker_eps_search(TensorDataset(preds), epsilons=(0.5, 0.0))
    with pytest.raises(NotImplementedError):
        modelpicker_eps_search(TensorDataset(torch.zeros(1025, 3, 2)))
    with pytest.raises(NotImplementedError):
        modelpicker_eps_search(TensorDataset(preds, n_global=60))
    if not torch.cuda.is_available():
        with pytest.raises(NotImplementedError, match="no CPU path"):
            modelpicker_eps_search(TensorDataset(preds), iterations=2, pool_size=5, budget=3)


def _dispatch_source():
    """The model_picker branch of main.py as the GPU tests' driver states it (tests/test_baselines.py)."""
    src = open(os.path.join(ROOT, "tests", "test_baselines.py")).read()
    return re.search(r"^def build\(dataset, args, loss_fn\):\n(?:    .*\n)+", src, flags=re.M).group(0)


def _run_dispatch(task, env_extra):
    code = (
        "import types\n"
        "import coda.baselines\n"
        "got = []\n"
        "class ModelPicker:\n"
        "    def __init__(self, dataset, epsilon=0.46):\n"
        "        got.append(epsilon)\n"
        "IID = ActiveTesting = VMA = Uncertainty = CODA = None\n"
        + _dispatch_source() +
        f"build(None, types.SimpleNamespace(method='model_picker', task={task!r}), None)\n"
        "from coda.baselines.modelpicker import TASK_EPS\n"
        "print('EPS', got[0], sorted(TASK_EPS.items()))\n")
    env = dict(os.environ, PYTHONPATH=ROOT, **env_extra)
    env.pop("CODA_REFERENCE_PATH", None)
    if not env_extra:
        env.pop("CODA_B200_TASK_EPS", None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr[-3000:]
    return r.stdout


def test_task_eps_file_reaches_main_py_dispatch(tmp_path):
    path = tmp_path / "best_epsilons.json"
    path.write_text(json.dumps({"taskA": {"best_avg": 0.41, "best_fast": 0.38},
                                "taskB.pt": {"best_avg": 0.37, "best_fast": 0.49}}))
    out = _run_dispatch("taskA", {"CODA_B200_TASK_EPS": str(path)})
    assert "not in TASK_EPS" not in out
    assert "EPS 0.41 [('taskA', 0.41), ('taskB', 0.37)]" in out
    out = _run_dispatch("taskB", {"CODA_B200_TASK_EPS": str(path)})
    assert "EPS 0.37" in out and "not in TASK_EPS" not in out
    out = _run_dispatch("taskA", {})                     # unset: the table stays empty, main.py's default
    assert "taskA not in TASK_EPS; using default" in out and "EPS 0.46 []" in out


def test_search_entry_points_are_declared_and_bound():
    from coda_b200 import _native as nat
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    arity = {"coda_b200_mp_runs_plan": 6, "coda_b200_mp_runs": 20, "coda_b200_majority": 5,
             "coda_b200_pool_accuracy": 8}
    for name, n in arity.items():
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
        assert m and len(m.group(1).split(",")) == n, name
        assert len(nat.SIGNATURES[name][1]) == n, name
    assert nat.VERSION == 203
    lib = nat.load()
    for name in arity:
        assert hasattr(lib, name)
