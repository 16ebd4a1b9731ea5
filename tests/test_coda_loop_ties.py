"""CODA's host-free loop with ``tie_rule="reference"`` on the GPU: isclose ties broken with the reference's
``random.choice`` draw, made on the device from a replica of Python's generator (csrc/pyrandom.cuh).  The generator
against the interpreter's, ``run_steps`` against the API loop on tie-heavy slabs, the trajectory goldens with ties,
interleaving and the refusals."""
import random
import types

import numpy as np
import pytest
import torch

from helpers import golden_names, golden_slab, load_golden
from test_coda_loop_ablations import _api_steps, _assert_same_state, _data, _dup_columns, _make

pytestmark = pytest.mark.gpu


def test_device_generator_matches_the_interpreter():
    from coda_b200 import _native as nat
    from coda_b200.selector import rng_state, rng_words, sample_setsize
    ops = []
    for n in (1, 2, 3, 4, 5, 64, 65, 1 << 20, (1 << 20) + 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1):
        ops += [(0, n, 0, 0)] * 150
    for m in (1, 5, 6, 7, 50, 333):
        s = sample_setsize(m)
        ops += [(1, s, m, s), (1, s + 1, m, s), (1, 3 * s, m, s)]
    ops += [(1, 2 ** 31 - 1, 40, sample_setsize(40))]
    random.seed(2024)
    for _ in range(100):
        random.random()
    st = random.getstate()
    want = []
    for kind, n, m, _s in ops:
        want += [random._inst._randbelow(n)] if kind == 0 else random.sample(range(n), m)
    dev = torch.device("cuda:0")
    state = rng_words(st).to(dev)
    opt = torch.tensor(ops, dtype=torch.int64, device=dev)
    out = torch.full((len(want),), -1, dtype=torch.int64, device=dev)
    nmax = max(n for k, n, m, s in ops if k == 1 and n <= s)
    pool = torch.zeros(nmax + 1, dtype=torch.int32, device=dev)
    seen = torch.zeros(2 ** 31 // 32, dtype=torch.int32, device=dev)          # the set branch's n < 2^31
    nat.call("coda_b200_pyrandom_run", state.data_ptr(), opt.data_ptr(), len(ops), out.data_ptr(), pool.data_ptr(),
             seen.data_ptr(), None)
    torch.cuda.synchronize()
    assert out.cpu().tolist() == want
    assert rng_state(state.cpu(), st[2]) == random.getstate()
    assert not seen.any()                                                     # the set branch leaves its bitmap clear


def _dup_data(copies=3, N=400):
    return _dup_columns(N=N, copies=copies)


KW = {"eig": {}, "uncertainty": dict(q="uncertainty")}


def _prefilter_kw(data):
    probe = _make(*data, {})
    d0 = sum(e.candidate_counts()[0] for e in probe.engines)
    probe.close()
    return dict(prefilter_n=d0 // 2)


def _ref_parity(kw, k, data, shards=None, record_best=True, seed=3):
    preds, labels = data
    random.seed(seed)
    api = _make(preds, labels, kw, shards)
    exp = _api_steps(api, labels, k)
    st = random.getstate()
    random.seed(seed)
    dev = _make(preds, labels, kw, shards)
    dev.run_steps(k, labels, record_best=record_best, tie_rule="reference")
    assert random.getstate() == st
    idx, q, tie = dev.history()
    assert idx.tolist() == exp[0]
    assert q.tobytes() == np.asarray(exp[1], np.float32).tobytes()
    assert tie.tolist() == exp[2]
    best, _ = dev.best_history()
    assert best.tolist() == (exp[3] if record_best else [-1] * k)
    _assert_same_state(dev, api)
    return exp


@pytest.mark.parametrize("record_best", [True, False])
@pytest.mark.parametrize("graph", ["1", "0"])
@pytest.mark.parametrize("shards", [1, 2, 3])
@pytest.mark.parametrize("kind", ["eig", "uncertainty", "prefilter"])
def test_reference_rule_equals_the_api_loop_on_exact_ties(kind, shards, graph, record_best, monkeypatch):
    """Three copies of every item: exact ties every step, their copies on different shards."""
    monkeypatch.setenv("CODA_B200_GRAPH", graph)
    data = _dup_data()
    kw = _prefilter_kw(data) if kind == "prefilter" else KW[kind]
    exp = _ref_parity(kw, 12, data, shards, record_best)
    assert sum(exp[2]) >= 3                                   # the reference drew among ties on several steps


def test_prefilter_ties_then_the_plain_arg_max():
    """Sampled steps with ties, then (n_s <= prefilter_n) the EIG loop's steps, from the same device stream."""
    data = _dup_data()
    probe = _make(*data, {})
    d0 = sum(e.candidate_counts()[0] for e in probe.engines)
    probe.close()
    exp = _ref_parity(dict(prefilter_n=d0 - 4), 10, data, shards=2)
    assert sum(exp[2][:4]) >= 1


def test_one_model_every_candidate_ties():
    """H = 1: no model disagrees, every unlabeled item is a candidate and every EIG is equal: 400 ties per step, above
    the API path's tie list."""
    from coda_b200.engine import TIE_CAP
    preds, labels = _data(H=1, N=400, C=5, seed=11)
    assert 400 > TIE_CAP
    exp = _ref_parity({}, 6, (preds, labels))
    assert exp[2] == [1] * 6


@pytest.mark.parametrize("kind", ["eig", "uncertainty", "prefilter"])
def test_api_device_api_interleaving(kind):
    data = _dup_data()
    preds, labels = data
    kw = _prefilter_kw(data) if kind == "prefilter" else KW[kind]
    random.seed(9)
    api = _make(preds, labels, kw)
    exp = _api_steps(api, labels, 9)
    st = random.getstate()
    random.seed(9)
    mix = _make(preds, labels, kw, shards=2)
    a = _api_steps(mix, labels, 2)
    mix.run_steps(5, labels, record_best=True, tie_rule="reference")
    b = _api_steps(mix, labels, 2)
    assert random.getstate() == st
    idx, q, tie = mix.history()
    assert idx.tolist() == exp[0][2:7] and tie.tolist() == exp[2][2:7]
    assert q.tobytes() == np.asarray(exp[1][2:7], np.float32).tobytes()
    assert a[0] + b[0] == exp[0][:2] + exp[0][7:]
    _assert_same_state(mix, api)


@pytest.mark.parametrize("name", golden_names())
def test_reference_rule_follows_every_trajectory_golden(name):
    """No skip for the goldens where the reference broke an isclose tie with random.choice: the loop equals the API loop
    from the goldens' seed, and both follow the golden wherever the device's EIG reproduces the reference's tie set.
    traj_h256 ties two items at 5.531311e-05 in the reference's fp32 EIG; the device scores them 4.4e-7 apart (inside
    the EIG parity budget, far outside isclose's 1e-8), so there both paths see one maximum and take it."""
    from coda_b200 import CODA, TensorDataset
    g = load_golden(name)
    preds, labels = golden_slab(g)
    K = int(g["steps"])
    random.seed(0)                                            # the goldens' seed (tests/golden/make_golden.py)
    api = CODA(TensorDataset(preds.cuda(), labels.cuda()), **g["ctor"])
    exp = _api_steps(api, labels, K)
    st = random.getstate()
    random.seed(0)
    sel = CODA(TensorDataset(preds.cuda(), labels.cuda()), **g["ctor"])
    sel.run_steps(K, labels, tie_rule="reference")
    idx, q, tie = sel.history()
    assert idx.tolist() == exp[0] and tie.tolist() == exp[2] and random.getstate() == st
    assert q.tobytes() == np.asarray(exp[1], np.float32).tobytes()
    ref_tie = (g["n_ties"][:K] > 1).astype(int)
    k = next((s for s in range(K) if idx[s] != g["idx"][s]), K)
    assert tie[:k].tolist() == ref_tie[:k].tolist()          # ties the device sees too: the reference's draws
    if k < K:                                                 # a reference tie the device's scores do not reproduce
        assert ref_tie[k] == 1 and tie[k] == 0
    if ref_tie[:k].any():
        assert sel.stochastic
    assert np.abs(q[:k].astype(np.float64) - g["q"][:k]).max(initial=0.0) < 5e-6


def test_refusals_raise_before_any_launch(monkeypatch):
    preds, labels = _data(N=200)
    random.seed(0)

    def refused(sel, exc, match):
        state = random.getstate()
        ctr = int(sel.engine.step_ctr.item())
        launches = sel.engine.counters["launches"]
        with pytest.raises(exc, match=match):
            sel.run_steps(3, labels, tie_rule="reference")
        assert random.getstate() == state and sel.engine.counters["launches"] == launches
        assert int(sel.engine.step_ctr.item()) == ctr and not sel.labeled_idxs
        assert getattr(sel.engine, "pyrng", None) is None

    for kw in ({}, dict(q="uncertainty"), dict(prefilter_n=5)):
        sel = _make(preds, labels, kw)
        sel.group = types.SimpleNamespace(world=2)
        refused(sel, NotImplementedError, "one process per GPU")
    sel = _make(preds, labels, {})
    monkeypatch.setattr(random, "_inst", random.SystemRandom())
    refused(sel, RuntimeError, "replaced")
    monkeypatch.undo()
    monkeypatch.setattr(random.Random, "_randbelow", lambda self, n: 0)
    refused(sel, RuntimeError, "_randbelow_with_getrandbits")
    monkeypatch.undo()
    sel.N = 2 ** 32
    refused(sel, NotImplementedError, "2\\*\\*32")
    sel.N = 200
    big = _make(preds, labels, dict(prefilter_n=150), shards=2)
    import coda_b200._native as nat
    monkeypatch.setattr(big.engine.lib, "coda_b200_pf_tie_max_m", lambda H: 100, raising=False)
    refused(big, NotImplementedError, "prefilter_n <= 100")
    monkeypatch.undo()
    with pytest.raises(ValueError, match="tie_rule"):
        sel.run_steps(1, labels, tie_rule="nope")
    assert nat.load().coda_b200_pf_tie_max_m(12) == 8 * (64 + 2 * 32)
