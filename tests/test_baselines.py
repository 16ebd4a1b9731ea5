"""The competing selectors (coda_b200.baselines) on the GPU against the reference's own runs on CPU
(tests/golden/baseline_*.npz and baselines_main_py.json, made by tests/golden/make_baseline_golden.py)."""
import hashlib
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN, ROOT

pytestmark = pytest.mark.gpu

sys.path.insert(0, GOLDEN)


def _digest(obj):
    return int.from_bytes(hashlib.sha256(obj).digest()[:8], "little", signed=True)


def _py_digest():
    return _digest(repr(random.getstate()).encode())


def _torch_digest():
    return _digest(torch.get_rng_state().numpy().tobytes())


def _seed_all():
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)


def _cases(method):
    names = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith(f"baseline_{method}_h") and f.endswith(".npz"))
    assert names, method
    return names


def _load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: z[k] for k in z.files}


def _setup(g, method):
    from coda.options import LOSS_FNS
    from coda_b200 import IID, VMA, ActiveTesting, ModelPicker, TensorDataset, Uncertainty
    from coda_b200.synth import synth
    preds, labels = synth(int(g["H"]), int(g["N"]), int(g["C"]), int(g["data_seed"]))
    assert np.array_equal(labels.numpy(), g["labels"])
    ds = TensorDataset(preds.cuda(), labels.cuda())
    _seed_all()
    cls = {"iid": IID, "uncertainty": Uncertainty, "activetesting": ActiveTesting, "vma": VMA}
    sel = ModelPicker(ds) if method == "model_picker" else cls[method](ds, LOSS_FNS["acc"])
    return sel, labels


@pytest.mark.parametrize("method", ["iid", "activetesting", "vma"])
def test_stochastic_baselines_follow_the_reference_draw_for_draw(method):
    for name in _cases(method):
        g = _load(name)
        sel, labels = _setup(g, method)
        if "score" in g:
            np.testing.assert_allclose(sel.score.cpu().numpy(), g["score"], rtol=1e-5, atol=1e-6)
        assert int(sel.get_best_model_prediction()) == int(g["best0"])
        for k in range(int(g["steps"])):
            idx, q = sel.get_next_item_to_label()
            assert isinstance(idx, int) and idx == int(g["idx"][k]), (name, k, idx, int(g["idx"][k]))
            np.testing.assert_allclose(q, g["q"][k], rtol=1e-5)
            sel.add_label(idx, int(labels[idx]), q)
            best = sel.get_best_model_prediction()
            assert isinstance(best, torch.Tensor) and best.dim() == 0
            assert int(best) == int(g["best"][k]), (name, k)
            assert _py_digest() == int(g["py"][k]) and _torch_digest() == int(g["torch"][k]), (name, k)
            if "lure" in g:
                np.testing.assert_allclose(sel.get_risk_estimates().cpu().numpy(), g["lure"][k], atol=1e-6)
        sel.close()


def test_uncertainty_follows_the_reference_while_its_maximum_is_separated():
    for name in _cases("uncertainty"):
        g = _load(name)
        sel, labels = _setup(g, "uncertainty")
        score = g["score"]
        np.testing.assert_allclose(sel.score.cpu().numpy(), score, atol=1e-6)
        assert sel.stochastic is False
        assert int(sel.get_best_model_prediction()) == int(g["best0"])      # main.py:84, a randperm over all H ties
        unl = np.ones(len(score), bool)
        for k in range(int(g["steps"])):
            top2 = np.sort(score[unl])[-2:]
            idx, q = sel.get_next_item_to_label()
            if top2[1] - top2[0] <= 1e-6:
                assert score[idx] >= top2[1] - 1e-6           # an equally good item, then the runs part ways
                break
            assert idx == int(g["idx"][k]) and abs(q - g["q"][k]) <= 1e-6, (name, k)
            sel.add_label(idx, int(labels[idx]), q)
            unl[idx] = False
            assert int(sel.get_best_model_prediction()) == int(g["best"][k])
            assert _torch_digest() == int(g["torch"][k]) and _py_digest() == int(g["py"][k])
        sel.close()


# The reference adds its C per-class terms into an fp32 running sum near log2 H (modelpicker.py:86).  The terms are
# nearly equal, so the roundings of the additions (up to half an ulp each) do not cancel: its values are off by up to
# C * ulp(log2 H) / 2 (2.4e-5 at H = 24, C = 100).  The kernel is checked to 1e-6 against an fp64 restatement of the
# same loop, and to that bound against the reference.
def _ref_tol(C, ent):
    return C * float(np.spacing(np.float32(np.nanmax(ent[np.isfinite(ent)])))) / 2 + 1e-6


def _fp64_entropies(hard, post, C, gamma, items):
    """modelpicker.py:74-86 in fp64 (with its 1e-12 clamp) for the given items."""
    post = post.astype(np.float64)
    hard = hard[items]
    out = np.zeros(len(items))
    for c in range(C):
        w = post[None, :] * np.where(hard == c, gamma, 1.0)
        p = np.maximum(w / w.sum(1, keepdims=True), 1e-12)
        out += -(p * np.log2(p)).sum(1) / C
    return out




def test_modelpicker_teacher_forced_on_the_reference_picks():
    for name in _cases("model_picker"):
        g = _load(name)
        sel, labels = _setup(g, "model_picker")
        hard = sel.hard.cpu().numpy().astype(np.int64) & 0xFFFF
        assert int(g["ties0"][sel.get_best_model_prediction()])
        for k in range(int(g["steps"])):
            ref = g["ent"][k]
            idx, q = sel.get_next_item_to_label()
            assert isinstance(idx, int) and q == 1.0 / (int(g["N"]) - k)
            ent = sel.entropies.cpu().numpy()
            unl = ~np.isnan(ref)
            assert np.array_equal(np.isinf(ent[unl]), np.isinf(ref[unl])), (name, k)
            fin = unl & np.isfinite(ref)
            tol = _ref_tol(int(g["C"]), ref)
            np.testing.assert_allclose(ent[fin], ref[fin], rtol=0, atol=tol)
            items = np.nonzero(fin)[0]
            exact = _fp64_entropies(hard, sel.posterior.cpu().numpy(), int(g["C"]), float(np.float32(sel.gamma)), items)
            np.testing.assert_allclose(ent[items], exact, rtol=0, atol=1e-6)
            assert ref[idx] <= np.nanmin(ref) + tol                 # our pick is a minimum under their entropies
            assert _torch_digest() == int(g["torch"][k]), (name, k)    # one randint per step, tie or not
            gi = int(g["idx"][k])
            sel.add_label(gi, int(labels[gi]), q)
            np.testing.assert_allclose(sel.posterior.cpu().numpy(), g["posterior"][k], rtol=1e-6, atol=1e-30)
            assert np.array_equal(sel.correct_counts.cpu().numpy(), g["counts"][k])
            best = sel.get_best_model_prediction()
            assert isinstance(best, int) and g["ties"][k][best], (name, k)   # drawn from the CUDA generator
        sel.close()


def test_modelpicker_free_running():
    for name in _cases("model_picker"):
        g = _load(name)
        sel, labels = _setup(g, "model_picker")
        sel.get_best_model_prediction()
        for k in range(int(g["steps"])):
            ref = g["ent"][k]
            idx, q = sel.get_next_item_to_label()
            m, tol = np.nanmin(ref), _ref_tol(int(g["C"]), ref)
            assert ref[idx] <= m + tol, (name, k)
            unique = np.sum(ref <= m + tol) == 1
            if idx != int(g["idx"][k]):
                assert not unique, (name, k)
                break
            sel.add_label(idx, int(labels[idx]), q)
            sel.get_best_model_prediction()
        sel.close()


def test_modelpicker_entropy_is_invariant_under_class_relabelling():
    """Items whose hard rows are equal up to a renaming of the classes get bit-identical entropies (the groups are
    summed in an order that does not depend on the class ids), at the uniform posterior and after labels."""
    from coda_b200 import ModelPicker, TensorDataset
    rng = np.random.default_rng(7)
    H, C, pairs = 40, 9, 64
    rows = rng.integers(0, 4, size=(pairs, H))
    rows[:, 0] = 0
    rows[:, 1] = 1                                           # every item has disagreement
    perm = np.stack([rng.permutation(C) for _ in range(pairs)])
    hard = np.concatenate([rows, np.take_along_axis(perm, rows, 1)], 0)          # item p and item pairs + p
    preds = np.full((H, 2 * pairs, C), 0.1 / (C - 1), np.float32)
    preds[np.arange(H)[:, None], np.arange(2 * pairs)[None, :], hard.T] = 0.9
    ds = TensorDataset(torch.from_numpy(preds).cuda(), torch.zeros(2 * pairs, dtype=torch.int64).cuda())
    torch.manual_seed(0)
    sel = ModelPicker(ds)
    for step in range(3):
        sel.get_next_item_to_label()
        e = sel.entropies.cpu().numpy()
        live = [p for p in range(pairs) if p not in sel.d_l_idxs and p + pairs not in sel.d_l_idxs]
        assert np.array_equal(e[live], e[[p + pairs for p in live]]), step
        sel.add_label(live[0], int(rng.integers(0, C)), 0.5)
    sel.close()


def test_selectors_reject_what_they_do_not_support():
    from coda_b200 import IID, ModelPicker, TensorDataset
    from coda_b200.synth import synth
    p, l = synth(4, 50, 3, 1)
    with pytest.raises(NotImplementedError, match="no CPU path"):
        ModelPicker(TensorDataset(p, l))
    with pytest.raises(NotImplementedError, match="shard"):
        IID(TensorDataset(p.cuda(), l, n_global=100), None)
    from coda.options import LOSS_FNS
    sel = IID(TensorDataset(p.cuda(), l.cuda()), LOSS_FNS["acc"])
    sel.add_label(3, 0, 0.1)
    with pytest.raises(ValueError):                          # list.remove of an item already labeled
        sel.add_label(3, 0, 0.1)
    sel.close()


_DRIVER = """\
import argparse
import os
import random

import mlflow
import numpy as np
import torch

from coda import CODA, Dataset, Oracle
from coda.baselines import IID, ActiveTesting, VMA, ModelPicker, Uncertainty
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


def build(dataset, args, loss_fn):
    simple = {"iid": IID, "uncertainty": Uncertainty, "activetesting": ActiveTesting, "vma": VMA}
    if args.method in simple:
        return simple[args.method](dataset, loss_fn)
    if args.method.startswith("coda"):
        return CODA.from_args(dataset, args)
    if args.method == "model_picker":
        from coda.baselines.modelpicker import TASK_EPS
        if args.task in TASK_EPS:
            return ModelPicker(dataset, epsilon=TASK_EPS[args.task])
        print(args.task, "not in TASK_EPS; using default")
        return ModelPicker(dataset)
    raise ValueError(args.method + " is not a supported method.")


def experiment(dataset, oracle, args, loss_fn, seed):
    reseed(seed)
    true_losses = oracle.true_losses(dataset.preds)
    best_loss = min(oracle.true_losses(dataset.preds))
    selector = build(dataset, args, loss_fn)
    best_model_idx_pred = selector.get_best_model_prediction()
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
device = torch.device("cuda" if torch.cuda.is_available() else "cpu")
print("device is", device)
dataset = Dataset(os.path.join(args.data_dir, args.task + ".pt"), device=device)
loss_fn = LOSS_FNS[args.loss]
oracle = Oracle(dataset, loss_fn=loss_fn)
name = args.experiment_name or args.task
mlflow.set_tracking_uri("sqlite:///coda.sqlite")
mlflow.set_experiment(name)
with mlflow.start_run(run_id=None, run_name=name + "-" + args.method):
    mlflow.log_params(vars(args))
    for seed in range(args.seeds):
        with mlflow.start_run(nested=True, run_id=None, run_name="%s-%s-%d" % (name, args.method, seed)):
            mlflow.log_param("seed", seed)
            stochastic = experiment(dataset, oracle, args, loss_fn, seed)
            mlflow.log_param("stochastic", stochastic)
        if not stochastic:
            break
"""


@pytest.mark.parametrize("method", ["iid", "uncertainty", "activetesting", "vma", "model_picker"])
def test_main_py_loop_matches_the_reference_run(tmp_path, method):
    import make_cfg1_golden as mk1
    from coda_b200.synth import synth
    gall = json.load(open(os.path.join(GOLDEN, "baselines_main_py.json")))
    g, task, iters = gall["methods"][method], gall["task"], gall["iters"]
    d = str(tmp_path)
    preds, labels = synth(task["H"], task["N"], task["C"], task["seed"])
    torch.save(preds, os.path.join(d, task["name"] + ".pt"))
    torch.save(labels, os.path.join(d, task["name"] + "_labels.pt"))
    with open(os.path.join(d, "driver.py"), "w") as f:
        f.write(_DRIVER)
    log = os.path.join(d, "mlflow.jsonl")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "stubs")]),
               MLFLOW_STUB_LOG=log, PYTHONSAFEPATH="1")
    env.pop("CODA_REFERENCE_PATH", None)
    cmd = [sys.executable, os.path.join(d, "driver.py"), "--task", task["name"], "--data-dir", d, "--method", method,
           "--seeds", "1", "--iters", str(iters)]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=d, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "device is cuda" in r.stdout
    out = mk1.parse_log(log)
    assert out["runs"] == g["runs"] and len(out["chosen_idx"]) == iters
    if method == "model_picker":
        assert "not in TASK_EPS; using default" in r.stdout
    # steps that are well conditioned: all of them for the draws, up to the first near-tie for the arg-extreme rules
    tol = {"uncertainty": 1e-6, "model_picker": 2e-6}.get(method)
    n = iters
    if tol is not None:
        n = next((k for k, gap in enumerate(g["gap"]) if gap <= tol), iters)
    assert out["chosen_idx"][:n] == g["chosen_idx"][:n], method
    assert out["true_class"][:n] == g["true_class"][:n]
    if method != "model_picker":             # ModelPicker draws its best model from the CUDA generator here
        assert out["best_model"][:n] == g["best_model"][:n]
        np.testing.assert_allclose(out["regret"][:n], g["regret"][:n], atol=1e-7)
        np.testing.assert_allclose(out["cumulative_regret"][:n], g["cumulative_regret"][:n], atol=1e-6)


@pytest.mark.parametrize("method", ["model_picker", "vma", "activetesting"])
def test_scale_256_models_500k_items(method):
    """The benchmark workload (a 51 GB slab), where the reference's VMA would need a 131 GB H x H x |D_U| tensor."""
    from coda.options import LOSS_FNS
    from coda_b200 import VMA, ActiveTesting, ModelPicker, SyntheticDataset
    ds = SyntheticDataset(256, 500_000, 100, seed=0, device="cuda")
    labels = ds.labels_host.numpy()
    _seed_all()
    sel = ModelPicker(ds) if method == "model_picker" else {"vma": VMA, "activetesting": ActiveTesting}[method](
        ds, LOSS_FNS["acc"])
    seen = set()
    for _ in range(20):
        idx, q = sel.get_next_item_to_label()
        assert 0 <= idx < 500_000 and idx not in seen and 0 < q <= 1
        seen.add(idx)
        sel.add_label(idx, int(labels[idx]), q)
        sel.get_best_model_prediction()
    assert int(sel.state.flags.item()) == 0
    assert int(sel.state.labeled.sum()) == 20
    sel.close()
    del ds
    torch.cuda.empty_cache()
