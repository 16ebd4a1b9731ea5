"""Checkpoint and resume of the competing selectors (``state_dict`` / ``load_state_dict``) on the GPU.  A run saved
after k1 steps, round-tripped through ``torch.save`` / ``torch.load`` and loaded into a new selector, continues for k2
steps exactly as the uninterrupted run of k1 + k2 steps does: the same picks, q bits and best models, ``stochastic``,
``history()`` / ``best_history()``, and the same Python, torch CPU and CUDA generator states afterwards.  Also across
layouts (shard counts, pieces, compact pieces, a 16-bit slab and its fp32 widening), and through a main.py-style
driver interrupted at step 40 of 100."""
import io
import json
import os
import random
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from helpers import ROOT

pytestmark = pytest.mark.gpu

METHODS = ["iid", "uncertainty", "activetesting", "vma", "model_picker"]
CLS = {"iid": "IID", "uncertainty": "Uncertainty", "activetesting": "ActiveTesting", "vma": "VMA",
       "model_picker": "ModelPicker"}
DEV = torch.device("cuda:0")


def _seed_all():
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    torch.cuda.manual_seed_all(0)


def _make(method, ds, eps=None, **kw):
    import coda_b200
    from coda.options import LOSS_FNS
    cls = getattr(coda_b200, CLS[method])
    if method == "model_picker":
        return cls(ds, **({} if eps is None else {"epsilon": eps}), **kw)
    return cls(ds, LOSS_FNS["acc"], **kw)


def _task(H=16, N=300, C=6, seed=7):
    from coda_b200.synth import synth
    return synth(H, N, C, seed)


def _layouts(preds, labels):
    """name -> (dataset factory, constructor keywords): the same slab values held in different layouts."""
    from coda_b200 import CompactSlab, TensorDataset
    from coda_b200.datasets import CompactDataset, ShardedCompactSlab, ShardedSlab
    from coda_b200.synth import shard_range
    N = preds.shape[1]
    lab = labels.to(DEV)
    halves = [shard_range(N, r, 2) for r in range(2)]
    whole = lambda: CompactSlab.from_dense(preds.to(DEV), 4)
    f16 = preds.half()
    return {
        "1": (lambda: TensorDataset(preds.to(DEV), lab), {}),
        "2": (lambda: TensorDataset(preds.to(DEV), lab), {"shards": 2}),
        "pieces": (lambda: TensorDataset(ShardedSlab([preds[:, lo:hi].contiguous().to(DEV) for lo, hi in halves]), lab),
                   {}),
        "compact": (lambda: CompactDataset(whole(), lab), {}),
        "compact_pieces": (lambda: CompactDataset(ShardedCompactSlab([whole().narrow_items(lo, hi).to(DEV)
                                                                      for lo, hi in halves]), lab), {}),
        "f16": (lambda: TensorDataset(f16.to(DEV), lab), {}),
        "f16_widened": (lambda: TensorDataset(f16.float().to(DEV), lab), {}),
    }


def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf)                      # torch's default: weights_only=True


def _part(sel, labels, k, how, trace, seed):
    """``k`` steps of main.py:91-94: ``how`` = "api", or run_steps under tie rule "philox" (with ``seed``) or
    "reference".  Appends (pick, q bits, best model) per step to ``trace``."""
    if how == "api":
        for _ in range(k):
            i, q = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), q)
            b = sel.get_best_model_prediction()
            trace.append((int(i), float(q).hex(), int(b)))
        return
    n0 = len(sel.history()[0])
    if how == "philox":
        assert sel.run_steps(k, labels, seed=seed) == k
    else:
        assert sel.run_steps(k, labels, tie_rule="reference") == k
    idx, q, _tie = sel.history()
    best, _bt = sel.best_history()
    trace += [(int(i), float(x).hex(), int(b)) for i, x, b in zip(idx[n0:], q[n0:], best[n0:])]


def _run(method, save, load, labels, k1, k2, first, second, *, resume, eps=None, before_save=None):
    """One run of k1 + k2 steps; with ``resume``, saved after k1 steps in layout ``save`` and continued in a new
    selector of layout ``load``.  -> everything the comparison reads."""
    _seed_all()
    sel = _make(method, save[0](), eps, **save[1])
    trace = []
    _part(sel, labels, k1, first, trace, seed=3)
    if before_save is not None:
        before_save(sel)
    if resume:
        sd = _roundtrip(sel.state_dict())
        sel.close()
        random.seed(1234)                        # the restore, not luck, must put the generators back
        torch.manual_seed(1234)
        torch.cuda.manual_seed_all(1234)
        sel = _make(method, load[0](), eps, **load[1])
        sel.load_state_dict(sd)
    _part(sel, labels, k2, second, trace, seed=5)
    idx, q, tie = sel.history()
    best, btie = sel.best_history()
    out = {"trace": trace, "stochastic": sel.stochastic,
           "hist": [idx.tolist(), [float(x).hex() for x in q], tie.tolist(), best.tolist(), btie.tolist()],
           "labeled": list(sel.d_l_idxs), "ys": list(sel.d_l_ys), "unlabeled": len(sel.d_u_idxs),
           "py": random.getstate(), "cpu": torch.get_rng_state(), "cuda": torch.cuda.get_rng_state(DEV)}
    sel.close()
    return out


def _same(a, b, where):
    for key in ("trace", "stochastic", "hist", "labeled", "ys", "unlabeled", "py"):
        assert a[key] == b[key], (where, key)
    assert torch.equal(a["cpu"], b["cpu"]), (where, "torch.get_rng_state()")
    assert torch.equal(a["cuda"], b["cuda"]), (where, "torch.cuda.get_rng_state()")


def _check(method, lay, save, load, labels, k1, k2, first, second, **kw):
    want = _run(method, lay[save], None, labels, k1, k2, first, second, resume=False, **kw)
    got = _run(method, lay[save], lay[load], labels, k1, k2, first, second, resume=True, **kw)
    assert len(want["trace"]) == k1 + k2
    _same(want, got, (method, save, load, k1, first, second))
    return want


@pytest.mark.parametrize("second", ["api", "philox", "reference"])
@pytest.mark.parametrize("first", ["api", "philox", "reference"])
@pytest.mark.parametrize("method", METHODS)
def test_resume_on_two_shards_equals_the_uninterrupted_run(method, first, second):
    preds, labels = _task()
    lay = _layouts(preds, labels)
    for k1 in (0, 1, 7):
        _check(method, lay, "1", "2", labels, k1, 12, first, second)


@pytest.mark.parametrize("save,load", [("2", "1"), ("1", "pieces"), ("compact", "compact_pieces"),
                                       ("f16", "f16_widened")])
@pytest.mark.parametrize("method", METHODS)
def test_resume_across_layouts(method, save, load):
    preds, labels = _task(seed=9)
    lay = _layouts(preds, labels)
    for first, second in (("api", "philox"), ("philox", "api"), ("reference", "reference"), ("philox", "philox")):
        _check(method, lay, save, load, labels, 7, 10, first, second)


@pytest.mark.parametrize("method", METHODS)
def test_resume_through_the_tie_paths_of_duplicated_items(method):
    """Every item four times over and every model twice: Uncertainty's item ties and the best-model ties are drawn on
    both sides of the split."""
    base, blab = _task(H=8, N=60, C=4, seed=5)
    preds = torch.cat([base, base], 0).repeat(1, 4, 1).contiguous()
    labels = blab.repeat(4)
    lay = _layouts(preds, labels)
    for first in ("api", "philox", "reference"):
        for second in ("api", "philox", "reference"):
            out = _check(method, lay, "1", "2", labels, 7, 12, first, second)
            assert out["stochastic"]
            if second != "api":
                assert any(out["hist"][4][-12:]), "no best-model tie after the split"
                if method == "uncertainty":
                    assert any(out["hist"][2][-12:]), "no item tie after the split"


def test_modelpicker_with_another_epsilon():
    preds, labels = _task(seed=11)
    lay = _layouts(preds, labels)
    for first, second in (("api", "api"), ("philox", "philox"), ("reference", "api"), ("api", "reference")):
        _check("model_picker", lay, "1", "2", labels, 7, 12, first, second, eps=0.3)
    _seed_all()
    sel = _make("model_picker", lay["1"][0](), 0.3)
    sel.run_steps(3, labels, seed=1)
    sd = _roundtrip(sel.state_dict())
    assert sd["epsilon"] == 0.3
    sel.close()
    other = _make("model_picker", lay["1"][0]())
    with pytest.raises(ValueError, match="epsilon"):
        other.load_state_dict(sd)
    assert other.d_l_idxs == [] and int(other.state.labeled.sum()) == 0
    other.close()


def test_activetesting_resume_keeps_the_items_removed_without_a_label():
    preds, labels = _task(seed=13)
    lay = _layouts(preds, labels)
    gone = []

    def remove_top(sel, n=3):
        score = sel.score.cpu().numpy().copy()
        for i in list(sel.d_l_idxs) + gone:
            score[i] = -np.inf
        for i in np.argsort(-score, kind="stable")[:n].tolist():
            sel.d_u_idxs.remove(i)
            gone.append(i)

    for first in ("api", "philox", "reference"):
        for second in ("api", "philox"):
            for k1 in (0, 7):
                want = got = None
                for resume in (False, True):
                    del gone[:]
                    out = _run("activetesting", lay["1"], lay["2"], labels, k1, 12, first, second, resume=resume,
                               before_save=remove_top)
                    if resume:
                        got = out
                    else:
                        want = out
                assert len(gone) == 3 and not set(gone) & set(want["labeled"])
                assert want["unlabeled"] == preds.shape[1] - len(want["labeled"]) - 3
                _same(want, got, (first, second, k1))


def test_one_process_per_gpu_and_foreign_states_are_refused_untouched():
    preds, labels = _task()
    lay = _layouts(preds, labels)
    _seed_all()
    sel = _make("vma", lay["1"][0]())
    sel.run_steps(5, labels, seed=1)
    sd = _roundtrip(sel.state_dict())
    sel.run_steps(3, labels, seed=1)                      # leaves 3 device steps not yet mirrored
    group = sel.group
    sel.group = types.SimpleNamespace(world=2)            # as built by one process per GPU (this process: one shard)
    mask = sel.state.labeled.clone()
    with pytest.raises(NotImplementedError, match="one process per GPU"):
        sel.state_dict()
    assert sel._loop_dirty and len(sel.d_l_idxs) == 5
    with pytest.raises(NotImplementedError, match="one process per GPU"):
        sel.load_state_dict(sd)
    assert sel._loop_dirty and len(sel.d_l_idxs) == 5 and torch.equal(sel.state.labeled, mask)
    sel.group = group
    assert len(sel.history()[0]) == 8
    sel.close()
    for method, foreign in (("activetesting", sd), ("vma", dict(sd, version=2)), ("vma", dict(sd, N=301))):
        fresh = _make(method, lay["1"][0]())
        py = random.getstate()
        with pytest.raises(ValueError):
            fresh.load_state_dict(foreign)
        assert fresh.d_l_idxs == [] and fresh.losses == [] and int(fresh.state.labeled.sum()) == 0
        assert random.getstate() == py
        fresh.close()


# ------------------------------------------------------------------------------------------------------------------
# a main.py-style driver (main.py:55-103), killed after step 40 of 100 and resumed from its checkpoint
# ------------------------------------------------------------------------------------------------------------------
_DRIVER = """\
import argparse
import os
import random

import mlflow
import numpy as np
import torch

from coda import Dataset, Oracle
from coda.baselines import IID, ActiveTesting, VMA, ModelPicker, Uncertainty
from coda.options import LOSS_FNS

ap = argparse.ArgumentParser()
ap.add_argument("--task")
ap.add_argument("--data-dir")
ap.add_argument("--method")
ap.add_argument("--iters", type=int, default=100)
ap.add_argument("--checkpoint", default="")
ap.add_argument("--stop-after", type=int, default=0)      # save the checkpoint after this step and exit
ap.add_argument("--resume", action="store_true")          # continue from the checkpoint
args = ap.parse_args()


def seed_all(seed):
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)


def build(dataset, loss_fn):
    simple = {"iid": IID, "uncertainty": Uncertainty, "activetesting": ActiveTesting, "vma": VMA}
    if args.method in simple:
        return simple[args.method](dataset, loss_fn)
    return ModelPicker(dataset)


device = torch.device("cuda")
dataset = Dataset(os.path.join(args.data_dir, args.task + ".pt"), device=device)
loss_fn = LOSS_FNS["acc"]
oracle = Oracle(dataset, loss_fn=loss_fn)
mlflow.set_tracking_uri("sqlite:///coda.sqlite")
mlflow.set_experiment(args.task)
with mlflow.start_run(run_id=None, run_name=args.task + "-" + args.method + "-0"):
    seed_all(0)
    true_losses = oracle.true_losses(dataset.preds)
    best_loss = min(oracle.true_losses(dataset.preds))
    selector = build(dataset, loss_fn)
    if args.resume:
        ckpt = torch.load(args.checkpoint)
        selector.load_state_dict(ckpt["selector"])
        first, total = ckpt["step"] + 1, ckpt["total"]
    else:
        best_model_idx_pred = selector.get_best_model_prediction()
        print("Regret at 0:", float(true_losses[best_model_idx_pred] - best_loss))
        first, total = 1, 0
    for step in range(first, args.iters + 1):
        chosen_idx, selection_prob = selector.get_next_item_to_label()
        true_class = oracle(chosen_idx)
        selector.add_label(chosen_idx, true_class, selection_prob)
        best_model_idx_pred = selector.get_best_model_prediction()
        regret = true_losses[best_model_idx_pred] - best_loss
        total += regret
        print("Regret at %d: %r %r" % (step, float(regret), float(total)))
        mlflow.log_metric("regret", float(regret), step=step)
        mlflow.log_metric("cumulative regret", float(total), step=step)
        if step == args.stop_after:
            torch.save({"selector": selector.state_dict(), "step": step, "total": float(total)}, args.checkpoint)
            break
    else:
        print("stochastic", selector.stochastic)
"""


def _driver(d, method, log, *extra):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "stubs")]),
               MLFLOW_STUB_LOG=log, PYTHONSAFEPATH="1")
    env.pop("CODA_REFERENCE_PATH", None)
    env.pop("CODA_B200_GPUS", None)
    cmd = [sys.executable, os.path.join(d, "driver.py"), "--task", "ckpt_task", "--data-dir", d, "--method", method,
           "--checkpoint", os.path.join(d, "ckpt.pt"), *extra]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=d, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return [ln for ln in r.stdout.splitlines() if ln.startswith(("Regret", "stochastic"))]


def _metrics(log):
    with open(log) as f:
        return [json.loads(ln) for ln in f if json.loads(ln)["kind"] == "log_metric"]


@pytest.mark.parametrize("method", METHODS)
def test_main_py_driver_interrupted_at_step_40_logs_the_same_regrets(tmp_path, method):
    d = str(tmp_path)
    preds, labels = _task(H=24, N=2000, C=10, seed=3)
    torch.save(preds, os.path.join(d, "ckpt_task.pt"))
    torch.save(labels, os.path.join(d, "ckpt_task_labels.pt"))
    with open(os.path.join(d, "driver.py"), "w") as f:
        f.write(_DRIVER)
    whole, parts = os.path.join(d, "whole.jsonl"), os.path.join(d, "parts.jsonl")
    want = _driver(d, method, whole)
    got = _driver(d, method, parts, "--stop-after", "40")
    assert len(got) == 41 and os.path.exists(os.path.join(d, "ckpt.pt"))
    got += _driver(d, method, parts, "--resume")
    assert len(want) == 102 and want[-1].startswith("stochastic")
    assert got == want
    m_want, m_got = _metrics(whole), _metrics(parts)
    assert len(m_want) == 200 and m_got == m_want
