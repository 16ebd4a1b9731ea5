"""BASELINE.json configs[0]: run the reference's REAL driver (its `main.py`, unmodified, with the
reference's own `coda` package) on the cifar10_5592 stand-in on CPU and keep what it logged.

    CODA_REFERENCE_PATH=<reference checkout> python tests/golden/make_cfg1_golden.py [iters]   # ~70 s per iteration on 8 cores

The paper's tensors are not in the reference checkout (README.md:31, a 3.25 GB download), so the task file is the
synthetic stand-in SURVEY.md 8(d) names: synth(80, 10000, 10, seed 0) saved as cifar10_5592.pt / _labels.pt.
MLflow is not installed: `tests/stubs/mlflow` records every call (parameters, nested runs, the per-step `regret`
and `cumulative regret` metrics of main.py:102-103) plus the loop's chosen_idx / best_model_idx_pred.
Output: tests/golden/cfg1_main_py.json.
"""
import json
import os
import subprocess
import sys
import tempfile

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ.get("CODA_REFERENCE_PATH", "")
TASK = dict(H=80, N=10000, C=10, seed=0)


def write_task(d):
    from coda_b200.synth import synth
    preds, labels = synth(TASK["H"], TASK["N"], TASK["C"], TASK["seed"])
    torch.save(preds, os.path.join(d, "cifar10_5592.pt"))
    torch.save(labels, os.path.join(d, "cifar10_5592_labels.pt"))


def run_main(main_py, data_dir, iters, log, pythonpath, extra_env=None, safe_path=False):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pythonpath), MLFLOW_STUB_LOG=log)
    if safe_path:
        env["PYTHONSAFEPATH"] = "1"
    env.update(extra_env or {})
    cmd = [sys.executable, main_py, "--task", "cifar10_5592", "--data-dir", data_dir, "--method", "coda", "--seeds", "1",
           "--iters", str(iters)]
    return subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=data_dir)


def parse_log(path):
    recs = [json.loads(l) for l in open(path)]
    out = {"regret": [], "cumulative_regret": [], "chosen_idx": [], "true_class": [], "best_model": [], "runs": [],
           "params": None, "seed_params": []}
    for r in recs:
        if r["kind"] == "log_metric" and r["key"] == "regret":
            out["regret"].append(r["value"]); out["chosen_idx"].append(r.get("chosen_idx"))
            out["true_class"].append(r.get("true_class")); out["best_model"].append(r.get("best_model_idx_pred"))
            assert r["step"] == len(out["regret"])
        elif r["kind"] == "log_metric" and r["key"] == "cumulative regret":
            out["cumulative_regret"].append(r["value"])
        elif r["kind"] == "start_run":
            out["runs"].append([r["run_name"], r["nested"]])
        elif r["kind"] == "log_params":
            out["params"] = r["params"]
        elif r["kind"] == "log_param":
            out["seed_params"].append([r["key"], r["value"]])
    return out


def reference_top(golden, k=12):
    """Second pass, in process: the reference's own `CODA` (imported from the reference checkout), teacher-forced along
    the trajectory main.py took, with the full EIG vector of every step reduced to its top-k candidates.  main.py does
    not log scores; index parity is ill-conditioned where two candidates are within fp32 noise (SURVEY.md 8c-3), and
    these values are what lets a test tell a near-tie from a wrong pick."""
    import random
    import types
    import numpy as np
    for name in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.path.insert(0, REF)
    for m in [m for m in sys.modules if m == "coda" or m.startswith("coda.")]:
        del sys.modules[m]
    import coda.coda as ref_coda
    assert ref_coda.__file__.startswith(REF)
    ref_coda.tqdm = lambda it, *a, **kw: it
    from coda_b200.synth import synth
    preds, labels = synth(TASK["H"], TASK["N"], TASK["C"], TASK["seed"])

    class DS:
        pass
    ds = DS()
    ds.preds, ds.labels, ds.device = preds, labels, preds.device
    random.seed(0); np.random.seed(0); torch.manual_seed(0)
    sel = ref_coda.CODA(ds)
    sel.get_best_model_prediction()
    top = []
    for i, idx in enumerate(golden["chosen_idx"]):
        q, cand = sel.eig_batched()
        order = torch.argsort(q, descending=True)[:k]
        top.append([[int(cand[j]), float(q[j])] for j in order.tolist()])
        assert int(cand[int(torch.argmax(q))]) == idx or abs(float(q.max()) - float(q[cand.index(idx)])) < 1e-7, (i, idx)
        sel.add_label(idx, int(labels[idx]), float(q[cand.index(idx)]))
        sel.get_best_model_prediction()
        print("step", i, "top2 gap", top[-1][0][1] - top[-1][1][1], flush=True)
    return top


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--top":
        path = os.path.join(HERE, "cfg1_main_py.json")
        g = json.load(open(path))
        g["top"] = reference_top(g)
        json.dump(g, open(path, "w"), indent=1)
        sys.exit(0)
    iters = int(sys.argv[1]) if len(sys.argv) > 1 else 25
    with tempfile.TemporaryDirectory() as d:
        write_task(d)
        log = os.path.join(d, "mlflow.jsonl")
        # sys.path[0] is the script's directory (the reference checkout): `coda` is the REFERENCE's package here
        r = run_main(os.path.join(REF, "main.py"), d, iters, log, [os.path.join(ROOT, "tests", "stubs")])
        if r.returncode != 0:
            sys.exit(r.stdout[-3000:] + r.stderr[-3000:])
        out = parse_log(log)
    out["task"] = TASK
    out["iters"] = iters
    out["stdout_head"] = r.stdout.splitlines()[:6]
    json.dump(out, open(os.path.join(HERE, "cfg1_main_py.json"), "w"), indent=1)
    print("cfg1 golden:", out["chosen_idx"], out["regret"])
