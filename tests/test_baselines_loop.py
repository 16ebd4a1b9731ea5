"""The competing selectors' host-free loop (``run_steps`` / ``history`` / ``best_history``) on the GPU, against the
reference goldens (tests/golden/baseline_*.npz), against the API path, and across layouts."""
import os
import random

import numpy as np
import pytest
import torch

from helpers import GOLDEN
from test_baselines_loop_host import tie_pick

pytestmark = pytest.mark.gpu

CLS = {"iid": "IID", "uncertainty": "Uncertainty", "activetesting": "ActiveTesting", "vma": "VMA",
       "model_picker": "ModelPicker"}


def _cases(method):
    return sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith(f"baseline_{method}_h") and f.endswith(".npz"))


def _load(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: z[k] for k in z.files}


def _py_digest():
    import hashlib
    return int.from_bytes(hashlib.sha256(repr(random.getstate()).encode()).digest()[:8], "little", signed=True)


def _seed_all():
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)


def _make(method, preds, labels, **kw):
    import coda_b200
    from coda.options import LOSS_FNS
    from coda_b200 import TensorDataset
    ds = TensorDataset(preds, labels)
    cls = getattr(coda_b200, CLS[method])
    return cls(ds, **kw) if method == "model_picker" else cls(ds, LOSS_FNS["acc"], **kw)


def _golden_selector(g, method, **kw):
    from coda_b200.synth import synth
    preds, labels = synth(int(g["H"]), int(g["N"]), int(g["C"]), int(g["data_seed"]))
    _seed_all()
    sel = _make(method, preds.cuda(), labels.cuda(), **kw)
    return sel, labels


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("method", ["iid", "activetesting", "vma"])
def test_device_loop_reproduces_the_reference_draw_for_draw(method, split):
    for name in _cases(method):
        g = _load(name)
        sel, labels = _golden_selector(g, method)
        assert int(sel.get_best_model_prediction()) == int(g["best0"])
        steps = int(g["steps"])
        parts = [1, 7, steps - 8] if split else [steps]
        for k in parts:
            assert sel.run_steps(k, labels, seed=5) == k
        idx, q, tie = sel.history()
        best, btie = sel.best_history()
        assert idx.tolist() == g["idx"].tolist(), name
        np.testing.assert_allclose(q, g["q"], rtol=1e-5)
        assert not tie.any()
        assert _py_digest() == int(g["py"][-1]), name
        for s in range(steps):
            assert g["ties"][s][best[s]], (name, s)
            if g["ties"][s].sum() == 1:
                assert best[s] == g["best"][s] and btie[s] == 0, (name, s)
        assert sel.d_l_idxs == g["idx"].tolist() and len(sel.d_u_idxs) == int(g["N"]) - steps
        if "lure" in g:
            assert sel.M == steps and len(sel.losses) == steps and len(sel.qs) == steps
            np.testing.assert_allclose(sel.get_risk_estimates().cpu().numpy(), g["lure"][-1], atol=1e-6)
        sel.close()


def test_uncertainty_device_loop_follows_the_reference_while_separated():
    for name in _cases("uncertainty"):
        g = _load(name)
        sel, labels = _golden_selector(g, "uncertainty")
        score = g["score"]
        sel.get_best_model_prediction()
        steps = int(g["steps"])
        sel.run_steps(steps, labels, seed=1)
        idx, q, _tie = sel.history()
        unl = np.ones(len(score), bool)
        for k in range(steps):
            top2 = np.sort(score[unl])[-2:]
            if top2[1] - top2[0] <= 1e-6:
                assert score[idx[k]] >= top2[1] - 1e-6
                break
            assert idx[k] == int(g["idx"][k]) and abs(q[k] - g["q"][k]) <= 1e-6, (name, k)
            unl[idx[k]] = False
        sel.close()


def test_modelpicker_device_loop_follows_the_reference_while_separated():
    from test_baselines import _ref_tol
    for name in _cases("model_picker"):
        g = _load(name)
        sel, labels = _golden_selector(g, "model_picker")
        sel.get_best_model_prediction()
        steps = int(g["steps"])
        sel.run_steps(steps, labels, seed=2)
        idx, q, _tie = sel.history()
        best, _bt = sel.best_history()
        for k in range(steps):
            ref = g["ent"][k]
            m, tol = np.nanmin(ref), _ref_tol(int(g["C"]), ref)
            assert ref[idx[k]] <= m + tol, (name, k)
            assert q[k] == 1.0 / (int(g["N"]) - k)
            if np.sum(ref <= m + tol) > 1 or idx[k] != int(g["idx"][k]):
                assert np.sum(ref <= m + tol) > 1, (name, k)
                break
        sel.close()


def test_modelpicker_teacher_forced_against_the_api_path():
    """Run the device loop one step at a time and replay each step through an API-path selector: the device pick is
    in the API entropies' minimum set, the posterior agrees to rtol 1e-6, the counts are equal and the best model is
    in the API's tie set, after every step."""
    from test_baselines import _ref_tol
    for name in _cases("model_picker"):
        g = _load(name)
        dev, labels = _golden_selector(g, "model_picker")
        api, _ = _golden_selector(g, "model_picker")
        for s in range(int(g["steps"])):
            dev.run_steps(1, labels, seed=3)
            idx, _q, _tie = dev.history()
            best, _bt = dev.best_history()
            i = int(idx[s])
            api.get_next_item_to_label()
            ent = api.entropies.cpu().numpy()
            fin = ent[np.isfinite(ent)]
            assert ent[i] <= fin.min() + _ref_tol(int(g["C"]), fin), (name, s)
            api.add_label(i, int(labels[i]), 0.5)
            np.testing.assert_allclose(dev.posterior.cpu().numpy(), api.posterior.cpu().numpy(), rtol=1e-6, atol=0)
            cc = api.correct_counts.cpu().numpy()
            assert np.array_equal(dev.correct_counts.cpu().numpy(), cc), (name, s)
            assert dev._n_disagree == api._n_disagree, (name, s)
            assert cc[best[s]] == cc.max(), (name, s)
        dev.close()
        api.close()


@pytest.mark.parametrize("method", ["iid", "activetesting", "vma"])
def test_mixed_api_and_device_steps_equal_a_pure_api_run(method):
    g = _load(_cases(method)[0])

    def api_steps(sel, labels, n, out):
        for _ in range(n):
            i, q = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), q)
            sel.get_best_model_prediction()
            out.append((i, q))

    ref, labels = _golden_selector(g, method)
    want = []
    api_steps(ref, labels, 30, want)
    py = random.getstate()
    ref.close()
    sel, labels = _golden_selector(g, method)
    got = []
    api_steps(sel, labels, 5, got)
    sel.run_steps(12, labels, seed=9)
    api_steps(sel, labels, 3, got)          # syncs the 12 device steps first
    idx, q, _ = sel.history()
    got = got[:5] + list(zip(idx.tolist(), q.tolist())) + got[5:]
    sel.run_steps(10, labels, seed=9)
    idx, q, _ = sel.history()
    got += list(zip(idx[12:].tolist(), q[12:].tolist()))
    assert [i for i, _ in got] == [i for i, _ in want]
    np.testing.assert_allclose([x for _, x in got], [x for _, x in want], rtol=1e-6)
    assert random.getstate() == py
    sel.close()


def _hist(sel):
    idx, q, tie = sel.history()
    best, btie = sel.best_history()
    return [a.tolist() for a in (idx, q, tie, best, btie)]


@pytest.mark.parametrize("method", ["iid", "uncertainty", "activetesting", "vma", "model_picker"])
def test_histories_are_identical_across_layouts(method, monkeypatch):
    from coda_b200.synth import synth
    preds, labels = synth(24, 400, 100, 11)
    out = {}
    for tag, kw, p, env in (("1", {}, preds, "1"), ("2", {"shards": 2}, preds, "1"), ("3", {"shards": 3}, preds, "1"),
                            ("eager", {}, preds, "0"), ("f16", {}, preds.half(), "1"),
                            ("bf16", {}, preds.bfloat16(), "1")):
        monkeypatch.setenv("CODA_B200_GRAPH", env)
        base = p.float() if p.dtype != torch.float32 else p
        _seed_all()
        if tag in ("f16", "bf16"):                       # against the fp32 widening of the same slab
            ref = _make(method, base.cuda(), labels.cuda())
            ref.run_steps(25, labels, seed=4)
            out[tag + "_ref"] = _hist(ref)
            ref.close()
            _seed_all()
        sel = _make(method, p.cuda(), labels.cuda(), **kw)
        sel.run_steps(25, labels, seed=4)
        out[tag] = _hist(sel)
        sel.close()
    for tag in ("2", "3", "eager"):
        assert out[tag] == out["1"], tag
    for tag in ("f16", "bf16"):
        assert out[tag] == out[tag + "_ref"], tag


def test_device_loop_from_a_compact_slab_equals_the_densified_slab():
    from coda_b200 import IID, CompactSlab, ModelPicker, TensorDataset, Uncertainty, VMA
    from coda.options import LOSS_FNS
    from coda_b200.synth import synth_compact
    ids, probs, labels = synth_compact(16, 300, 20, 4, seed=5)
    cs = CompactSlab(ids, probs, 20).to(torch.device("cuda:0"))
    dense = cs.densify()
    for cls in (IID, Uncertainty, VMA, ModelPicker):
        hs = []
        for p in (cs, dense):
            _seed_all()
            sel = cls(TensorDataset(p, labels.cuda())) if cls is ModelPicker else cls(TensorDataset(p, labels.cuda()),
                                                                                        LOSS_FNS["acc"])
            sel.run_steps(20, labels, seed=8)
            hs.append(_hist(sel))
            sel.close()
        # q of Uncertainty (its entropy) and of AT / VMA (their normalised scores) derive from the ensemble sums, which
        # the compact scan adds in another order (the API path alike): picks, ties and best models are identical
        np.testing.assert_allclose(hs[0][1], hs[1][1], rtol=1e-6)
        assert hs[0][:1] + hs[0][2:] == hs[1][:1] + hs[1][2:], cls.__name__


def test_tie_draws_follow_the_philox_model():
    """Duplicated items and duplicated models: every model predicts the same class on every item, so every unlabeled
    item ties for Uncertainty's maximum and for ModelPicker's minimum (no item has disagreement), and every model ties
    for the best one.  The device's item and best-model draws are the NumPy Philox model's (item: label count before
    the step, purpose 0; best model: label count after it, purpose 1).  IID draws its items from Python random; its
    best-model ties follow the same stream."""
    H, N, C = 6, 64, 3
    preds = torch.full((H, N, C), 0.2)
    preds[:, :, 0] = 0.6
    labels = torch.zeros(N, dtype=torch.int64)
    for method in ("uncertainty", "model_picker", "iid"):
        for seed in (1, 77):
            _seed_all()
            sel = _make(method, preds.cuda(), labels.cuda())
            sel.run_steps(10, labels, seed=seed)
            idx, _q, tie = sel.history()
            best, btie = sel.best_history()
            unl = list(range(N))
            for s in range(10):
                if method != "iid":
                    want = unl[tie_pick(seed, s, 0, len(unl))]
                    assert idx[s] == want and tie[s] == 1, (method, seed, s)
                unl.remove(int(idx[s]))
                assert best[s] == tie_pick(seed, s + 1, 1, H) and btie[s] == 1, (method, seed, s)
            assert sel.stochastic
            sel.close()


def test_vma_stop_hands_over_to_the_api_path():
    """Only the first j items have disagreeing models: after j labels VMA's weights are all 0 and vma.py falls back to
    random.choice; run_steps finishes on the API path with the same picks and Python state as a pure API run."""
    H, N, C, j = 8, 120, 4, 6
    g = torch.Generator().manual_seed(0)
    preds = torch.full((H, N, C), 0.1)
    preds[:, :, 0] = 0.7
    for n in range(j):                                   # two of the eight models disagree on items 0 .. j-1
        preds[H - 2:, n, 0] = 0.1
        preds[H - 2:, n, 1] = 0.7
    labels = torch.randint(0, C, (N,), generator=g)
    _seed_all()
    ref = _make("vma", preds.cuda(), labels.cuda())
    want = []
    for _ in range(15):
        i, q = ref.get_next_item_to_label()
        ref.add_label(i, int(labels[i]), q)
        ref.get_best_model_prediction()
        want.append(i)
    py = random.getstate()
    ref.close()
    _seed_all()
    sel = _make("vma", preds.cuda(), labels.cuda())
    assert sel.run_steps(15, labels, seed=0) == 15
    idx, _q, _t = sel.history()
    assert len(idx) == j and sorted(idx.tolist()) == list(range(j))
    assert sel.d_l_idxs == want
    assert random.getstate() == py
    sel.close()


def test_device_loop_rejects_what_it_does_not_run():
    from coda_b200.synth import synth
    preds, labels = synth(4, 50, 3, 1)
    sel = _make("iid", preds.cuda(), labels.cuda())
    with pytest.raises(ValueError):
        sel.run_steps(51, labels)
    with pytest.raises(ValueError):
        sel.run_steps(3, labels[:10])
    sel.loss_fn = lambda p, l, **kw: torch.zeros(p.shape[0])
    with pytest.raises(NotImplementedError, match="API loop"):
        sel.run_steps(3, labels)
    sel.close()


def _coda_goldens():
    from helpers import golden_names
    return golden_names()


@pytest.mark.parametrize("name", _coda_goldens())
def test_coda_best_history_equals_the_api_best_model_per_step(name):
    """CODA.run_steps(..., record_best=True) records get_best_model_prediction() of every step: teacher-forced through
    the API path on the device loop's own picks, on every trajectory golden the device-loop test uses.  A step run on
    the default graph records nothing (-1)."""
    from helpers import golden_slab, load_golden
    from coda_b200 import CODA, TensorDataset
    g = load_golden(name)
    if int(g["n_ties"].max()) > 1:
        pytest.skip("the reference broke an isclose tie with random.choice on this golden")
    preds, labels = golden_slab(g)
    K = int(g["steps"])
    mk = lambda: CODA(TensorDataset(preds.cuda(), labels.cuda()), **g["ctor"])
    dev = mk()
    dev.run_steps(1, labels)
    dev.run_steps(K - 1, labels, record_best=True)
    idx, q, _tie = dev.history()
    best, btie = dev.best_history()
    assert len(best) == K and best[0] == -1 and not btie.any()
    assert idx.tolist() == g["idx"].tolist()
    api = mk()
    for s in range(K):
        api.add_label(int(idx[s]), int(labels[int(idx[s])]), float(q[s]))
        b = int(api.get_best_model_prediction())
        assert b == int(g["best_model"][s]), (name, s)
        if s:
            assert best[s] == b, (name, s)
    dev.close()
    api.close()
