"""Golden fixtures for the competing selectors, made by RUNNING THE REFERENCE (CPU, fp32).

    CODA_REFERENCE_PATH=<reference checkout> python tests/golden/make_baseline_golden.py [per_method] [main_py]

per_method -> tests/golden/baseline_<method>_h<H>_n<N>_c<C>.npz: the reference's class on a seeded synthetic slab
(``coda_b200.synth``), free-running the main.py loop (main.py:84-94) from ``seed_all(0)``.  Per step: the pick and q,
digests of the Python ``random`` state and of ``torch.get_rng_state()`` after the step, the best model and its tie
set; per method: the static scores (Uncertainty, ActiveTesting, VMA), the entropy vector of every step with NaN at
labeled items (ModelPicker), the posterior and counts (ModelPicker), the LURE risks (ActiveTesting, VMA).
ModelPicker draws its best model with ``device=self.device`` (modelpicker.py:106, 109), i.e. from the CUDA generator on
a GPU; here the CPU generator's state is restored around that call so that the recorded CPU stream is the one a GPU
run sees.

main_py -> tests/golden/baselines_main_py.json: the reference's real ``main.py`` for each of the five methods, one seed,
100 iterations, with the recording MLflow stub (tests/stubs/mlflow), on the cfg1 task tensors (make_cfg1_golden.TASK)
written under a task name that is not in the reference's ModelPicker epsilon table, so both sides use epsilon = 0.46.
Per method also the gap between the reference's best and second-best score at every step along its own trajectory
(Uncertainty, ModelPicker): where it is within fp32 noise the pick is ill-conditioned.
"""
import hashlib
import json
import os
import random
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import make_cfg1_golden as mk1  # noqa: E402
import make_golden as mk  # noqa: E402

CASES = [  # (H, N, C, data seed, steps, methods)
    (12, 500, 6, 1, 40, ("iid", "uncertainty", "activetesting", "vma", "model_picker")),
    (24, 400, 100, 2, 40, ("iid", "uncertainty", "activetesting", "vma", "model_picker")),
    (256, 1500, 100, 3, 15, ("activetesting", "vma", "model_picker")),
]
MAIN_TASK = "cfg1_baselines"
METHODS = ("iid", "uncertainty", "activetesting", "vma", "model_picker")


def digest(obj):
    return int.from_bytes(hashlib.sha256(obj).digest()[:8], "little", signed=True)


def py_digest():
    return digest(repr(random.getstate()).encode())


def torch_digest():
    return digest(torch.get_rng_state().numpy().tobytes())


def ref_classes():
    mk.import_reference()
    import coda.baselines as rb
    assert rb.__file__.startswith(mk.REF), rb.__file__
    from coda.options import LOSS_FNS
    return rb, LOSS_FNS["acc"]


def make(rb, loss, method, ds):
    return {"iid": lambda: rb.IID(ds, loss), "uncertainty": lambda: rb.Uncertainty(ds, loss),
            "activetesting": lambda: rb.ActiveTesting(ds, loss), "vma": lambda: rb.VMA(ds, loss),
            "model_picker": lambda: rb.ModelPicker(ds)}[method]()


def static_scores(method, preds):
    """The reference's per-item score over all items (uncertainty.py:6-11, activetesting.py:33-44, vma.py:18-41)."""
    import coda.baselines.uncertainty as ru
    H, N, _ = preds.shape
    if method == "uncertainty":
        return ru.uncertainty(preds, list(range(N))).numpy()
    losses = 1 - preds.mean(dim=0)[torch.arange(N).unsqueeze(0), preds.argmax(dim=2)]      # (H, N)
    if method == "activetesting":
        return losses.sum(dim=0).numpy()
    out = torch.zeros(N)
    iu = torch.triu_indices(H, H, offset=1)
    for lo in range(0, N, 256):
        l = losses[:, lo:lo + 256]
        out[lo:lo + 256] = (l.unsqueeze(0) - l.unsqueeze(1)).abs()[iu[0], iu[1]].sum(dim=0)
    return out.numpy()


def best_with_ties(sel, method):
    if method == "model_picker":
        state = torch.get_rng_state()
        best = int(sel.get_best_model_prediction())
        torch.set_rng_state(state)                        # the GPU run draws this from the CUDA generator
        c = sel.correct_counts
        ties = np.arange(sel.H) if not sel.d_l_idxs else torch.nonzero(c == c.max()).flatten().numpy()
        return best, ties
    labeled = len(sel.d_l_idxs) > 0
    if method in ("activetesting", "vma") and not labeled:
        return int(sel.get_best_model_prediction()), np.arange(sel.H)
    risk = sel.get_risk_estimates()
    best = int(sel.get_best_model_prediction())
    return best, torch.nonzero(risk == risk.min()).flatten().numpy()


def run_case(rb, loss, method, H, N, C, seed, steps):
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, seed)
    ds = mk._DS(preds, labels)
    mk.seed_all(0)
    sel = make(rb, loss, method, ds)
    out = {"H": H, "N": N, "C": C, "data_seed": seed, "steps": steps}
    if method != "model_picker" and method != "iid":
        out["score"] = static_scores(method, preds).astype(np.float32)
    best0, ties0 = best_with_ties(sel, method)
    rec = {k: [] for k in ("idx", "q", "py", "torch", "best", "ties", "ent", "posterior", "counts", "lure")}
    for _ in range(steps):
        if method == "model_picker":
            ent = np.full(N, np.nan, np.float32)
            u = list(sel.d_u_idxs)
            hard = preds.argmax(dim=2).transpose(0, 1)
            e = sel.compute_entropies(hard[u], sel.posterior, H, C, sel.gamma)
            m = sel._disagreement_mask[u]
            if m.any():
                e = e.clone()
                e[~m] = float("inf")
            ent[u] = e.numpy()
            rec["ent"].append(ent)
        idx, q = sel.get_next_item_to_label()
        idx = int(idx)
        sel.add_label(idx, int(labels[idx]), q)
        best, ties = best_with_ties(sel, method)
        rec["idx"].append(idx); rec["q"].append(float(q)); rec["best"].append(best)
        t = np.zeros(H, bool); t[ties] = True
        rec["ties"].append(t)
        rec["py"].append(py_digest()); rec["torch"].append(torch_digest())
        if method == "model_picker":
            rec["posterior"].append(sel.posterior.numpy().copy()); rec["counts"].append(sel.correct_counts.numpy().copy())
        if method in ("activetesting", "vma"):
            rec["lure"].append(sel.get_risk_estimates().numpy().copy())
    out.update(best0=best0, ties0=np.isin(np.arange(H), ties0), labels=labels.numpy())
    for k, v in rec.items():
        if v:
            out[k] = np.asarray(v)
    out["q"] = np.asarray(rec["q"], np.float64)
    name = f"baseline_{method}_h{H}_n{N}_c{C}"
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print(name, "picks", rec["idx"][:10], flush=True)


def score_gaps(rb, loss, method, preds, labels, picks):
    """Second-best minus best score of the reference at every step of its own trajectory (maximum for Uncertainty,
    minimum for ModelPicker), with the draws the selection loop would make replayed from main.py's seed."""
    ds = mk._DS(preds, labels)
    mk.seed_all(0)
    sel = make(rb, loss, method, ds)
    H, N, C = preds.shape
    gaps = []
    if method == "uncertainty":
        s = torch.from_numpy(static_scores(method, preds))
    hard = preds.argmax(dim=2).transpose(0, 1)
    for idx in picks:
        u = list(sel.d_u_idxs)
        if method == "uncertainty":
            v = -s[u]
        else:
            v = sel.compute_entropies(hard[u], sel.posterior, H, C, sel.gamma)
            m = sel._disagreement_mask[u]
            if m.any():
                v = v.clone()
                v[~m] = float("inf")
        two = torch.topk(v, 2, largest=False).values
        gaps.append(float(two[1] - two[0]))
        sel.add_label(idx, int(labels[idx]), 0.5)
    return gaps


def main_py_goldens(rb, loss, iters=100):
    from coda_b200.synth import synth
    t = mk1.TASK
    preds, labels = synth(t["H"], t["N"], t["C"], t["seed"])
    out = {"task": dict(t, name=MAIN_TASK), "iters": iters, "methods": {}}
    with tempfile.TemporaryDirectory() as d:
        torch.save(preds, os.path.join(d, MAIN_TASK + ".pt"))
        torch.save(labels, os.path.join(d, MAIN_TASK + "_labels.pt"))
        for method in METHODS:
            log = os.path.join(d, method + ".jsonl")
            env = dict(os.environ, PYTHONPATH=os.path.join(ROOT, "tests", "stubs"), MLFLOW_STUB_LOG=log)
            cmd = [sys.executable, os.path.join(mk.REF, "main.py"), "--task", MAIN_TASK, "--data-dir", d, "--method",
                   method, "--seeds", "1", "--iters", str(iters)]
            import subprocess
            r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=d)
            if r.returncode != 0:
                sys.exit(r.stdout[-3000:] + r.stderr[-3000:])
            g = mk1.parse_log(log)
            if method in ("uncertainty", "model_picker"):
                g["gap"] = score_gaps(rb, loss, method, preds, labels, g["chosen_idx"])
            out["methods"][method] = g
            print(method, g["chosen_idx"][:8], flush=True)
    json.dump(out, open(os.path.join(HERE, "baselines_main_py.json"), "w"))


if __name__ == "__main__":
    what = sys.argv[1:] or ["per_method", "main_py"]
    rb, loss = ref_classes()
    if "per_method" in what:
        for H, N, C, seed, steps, methods in CASES:
            for method in methods:
                run_case(rb, loss, method, H, N, C, seed, steps)
    if "main_py" in what:
        main_py_goldens(rb, loss)
