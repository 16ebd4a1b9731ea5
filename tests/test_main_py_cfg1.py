"""BASELINE.json configs[0] / north_star "main.py and the MLflow logging run unchanged": the reference driver's
experiment loop, executed as a subprocess against THIS package on the GPU with a recording MLflow stand-in
(`tests/stubs/mlflow`; MLflow is not installed in the images), compared with what the reference's real `main.py` logged
when it ran on the reference's own `coda` package on CPU (`tests/golden/cfg1_main_py.json`, made by
`tests/golden/make_cfg1_golden.py`).

Reference sources are never copied into this repository, so the driver is written here: it takes main.py's command
line and defaults (main.py:28-53), seeds every RNG as main.py:19-26 does, loads the task through `coda.datasets.Dataset`
/ `coda.oracle.Oracle` / `coda.options.LOSS_FNS` (main.py:110-118), opens the experiment run and the nested seed run
with their parameters (main.py:132-164), and runs the selection loop with its regret metrics (main.py:55-105) -- the
same calls, in the same order, with the same RNG consumption.
"""
import json
import os
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

sys.path.insert(0, GOLDEN)

_DRIVER = """\
import argparse
import os
import random

import mlflow
import numpy as np
import torch

from coda import CODA, Dataset, Oracle
from coda.options import LOSS_FNS


def command_line():
    ap = argparse.ArgumentParser()
    for flag, default, kind in (("--task", None, str), ("--data-dir", "data", str), ("--iters", 100, int),
                                ("--seeds", 5, int), ("--experiment-name", None, str), ("--loss", "acc", str),
                                ("--method", "iid", str), ("--alpha", 0.9, float), ("--learning-rate", 0.01, float),
                                ("--multiplier", 2.0, float), ("--prefilter-n", 0, int), ("--q", "eig", str)):
        ap.add_argument(flag, default=default, type=kind)
    for flag in ("--force-rerun", "--no-mlflow", "--no-diag-prior"):
        ap.add_argument(flag, action="store_true")
    return ap.parse_args()


def reseed(seed):
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)


def experiment(dataset, oracle, args, seed):
    reseed(seed)
    true_losses = oracle.true_losses(dataset.preds)
    best_loss = min(oracle.true_losses(dataset.preds))
    print("Best possible loss is", best_loss)
    selector = CODA.from_args(dataset, args)
    best_model_idx_pred = selector.get_best_model_prediction()
    print("Regret at 0:", true_losses[best_model_idx_pred] - best_loss)
    total = 0
    for step in range(1, args.iters + 1):
        chosen_idx, selection_prob = selector.get_next_item_to_label()
        true_class = oracle(chosen_idx)
        selector.add_label(chosen_idx, true_class, selection_prob)
        best_model_idx_pred = selector.get_best_model_prediction()
        regret = true_losses[best_model_idx_pred] - best_loss
        total += regret
        mlflow.log_metric("regret", float(regret), step=step)        # the stub also records this frame's pick
        mlflow.log_metric("cumulative regret", float(total), step=step)
    return selector.stochastic


args = command_line()
assert args.method == "coda" and not args.no_mlflow
device = torch.device("cuda" if torch.cuda.is_available() else "cpu")
print("device is", device)
dataset = Dataset(os.path.join(args.data_dir, args.task + ".pt"), device=device)
oracle = Oracle(dataset, loss_fn=LOSS_FNS[args.loss])
name = args.experiment_name or args.task
mlflow.set_tracking_uri("sqlite:///coda.sqlite")
mlflow.set_experiment(name)
with mlflow.start_run(run_id=None, run_name=name + "-" + args.method):
    mlflow.log_params(vars(args))
    for seed in range(args.seeds):
        with mlflow.start_run(nested=True, run_id=None, run_name="%s-%s-%d" % (name, args.method, seed)):
            mlflow.log_param("seed", seed)
            stochastic = experiment(dataset, oracle, args, seed)
            mlflow.log_param("stochastic", stochastic)
        if not stochastic:
            break
"""


def _run(tmp_path, extra_env=None, iters=None):
    import make_cfg1_golden as mk
    g = json.load(open(os.path.join(GOLDEN, "cfg1_main_py.json")))
    iters = iters or g["iters"]
    d = str(tmp_path)
    mk.write_task(d)
    driver = os.path.join(d, "driver.py")
    with open(driver, "w") as f:
        f.write(_DRIVER)
    log = os.path.join(d, "mlflow.jsonl")
    # PYTHONSAFEPATH keeps the driver's directory off sys.path: `coda` resolves to this repository's shim
    r = mk.run_main(driver, d, iters, log, [ROOT, os.path.join(ROOT, "tests", "stubs")], extra_env=extra_env, safe_path=True)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = mk.parse_log(log)
    return g, out, r.stdout


def _compare(g, out, stdout, iters):
    assert "device is cuda" in stdout and "Loaded preds of shape torch.Size([80, 10000, 10])" in stdout
    # MLflow plumbing of main.py:132-164: experiment run + nested seed run, parameters, per-step metrics
    assert out["runs"] == g["runs"] == [["cifar10_5592-coda", False], ["cifar10_5592-coda-0", True]]
    assert out["params"]["method"] == "coda" and out["params"]["task"] == "cifar10_5592"
    assert ["seed", 0] in out["seed_params"] and "stochastic" in [k for k, _ in out["seed_params"]]
    assert len(out["regret"]) == len(out["cumulative_regret"]) == len(out["chosen_idx"]) == iters
    # the selection trajectory (main.py:91-103): items, revealed classes, predicted best model, regret.  Free-running
    # index parity is ill-conditioned where the reference's own top candidates are within fp32 noise (SURVEY.md 8c-3):
    # the trajectories must be identical up to the first such step, and there our pick must be epsilon-optimal under
    # the REFERENCE's scores (golden["top"]: the reference's top candidates of every step along its trajectory).
    ref_idx = g["chosen_idx"][:iters]
    same = 0
    while same < iters and out["chosen_idx"][same] == ref_idx[same]:
        same += 1
    assert out["true_class"][:same] == g["true_class"][:same]
    assert out["best_model"][:same] == g["best_model"][:same]
    np.testing.assert_allclose(out["regret"][:same], g["regret"][:same], atol=1e-7)
    np.testing.assert_allclose(out["cumulative_regret"][:same], g["cumulative_regret"][:same], atol=1e-6)
    if same < iters:
        assert "top" in g, "golden has no reference scores to judge the divergence at step %d" % same
        top = dict((int(i), float(v)) for i, v in g["top"][same])
        best = max(top.values())
        ours = out["chosen_idx"][same]
        assert ours in top and top[ours] >= best - 5e-6, (same, ours, g["top"][same][:4])
        assert top[ref_idx[same]] >= best - 5e-6
    return same


def test_reference_main_py_runs_unchanged_on_one_gpu(tmp_path):
    """The driver loop on one GPU, all golden steps."""
    g, out, stdout = _run(tmp_path)
    keep = os.environ.get("CODA_B200_KEEP_MAIN_LOG")
    if keep:
        with open(keep, "w") as f:
            f.write(stdout[-6000:])
            f.write("\n--- mlflow stub log (parsed) ---\n" + json.dumps(out)[:4000] + "\n")
    same = _compare(g, out, stdout, g["iters"])
    if keep:
        with open(keep, "a") as f:
            f.write("identical to the reference's CPU run of the same driver for the first %d of %d steps\n" % (same, g["iters"]))


def test_reference_main_py_runs_unchanged_on_all_gpus(tmp_path):
    """Same driver, same command line; CODA_B200_GPUS in the environment makes the selector shard the slab over the
    GPUs of the box from inside the one process main.py starts (SURVEY.md 8e process model)."""
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    g, out, stdout = _run(tmp_path, extra_env={"CODA_B200_GPUS": str(min(n, 8))}, iters=10)
    _compare(g, out, stdout, 10)
