"""CODA's host-free loop with the acquisitions other than EIG (``q='iid'``, ``q='uncertainty'``, ``prefilter_n``) on the
GPU: ``run_steps`` against the API loop (get_next_item_to_label -> add_label -> get_best_model_prediction) from the same
state, against the reference goldens (tests/golden/acquisitions.json), across the candidate-set boundaries, pre-draw
chunks, ties, interleaving, slab formats and the refusals."""
import json
import random
import types

import numpy as np
import pytest
import torch

from helpers import GOLDEN

pytestmark = pytest.mark.gpu

KINDS = {"iid": dict(q="iid"), "uncertainty": dict(q="uncertainty"), "prefilter": dict(prefilter_n=50)}


def _data(H=12, N=600, C=6, seed=17, disagree=None):
    """synth data; with ``disagree`` only the first ``disagree`` items can have models that disagree (on the others
    every model's scores are pulled halfway to model 0's class, which keeps them distinct), so the candidate set runs
    out within a short run."""
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, seed=seed)
    if disagree is not None:
        rest = preds[:, disagree:]
        onehot = torch.nn.functional.one_hot(rest[0].argmax(-1), C).to(preds.dtype)
        preds[:, disagree:] = 0.5 * rest + 0.5 * onehot
    return preds, labels


def _make(preds, labels, kw, shards=None, device="cuda:0"):
    from coda_b200 import CODA, TensorDataset
    return CODA(TensorDataset(preds.to(device), labels.to(device)), shards=shards, **kw)


class _ChoiceCounter:
    """Counts the random.choice calls of one API step: the steps where the reference draws among isclose ties."""

    def __enter__(self):
        self.orig, self.n = random.choice, 0

        def choice(seq):
            self.n += 1
            return self.orig(seq)
        random.choice = choice
        return self

    def __exit__(self, *a):
        random.choice = self.orig


def _api_steps(sel, labels, k):
    idx, q, tie, best = [], [], [], []
    for _ in range(k):
        with _ChoiceCounter() as cc:
            i, qq = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), qq)
        best.append(int(sel.get_best_model_prediction()))
        idx.append(int(i)); q.append(qq); tie.append(1 if cc.n else 0)
    return idx, q, tie, best


def _assert_same_state(dev, api):
    assert dev.stochastic == api.stochastic
    assert torch.equal(dev.dirichlets.cpu(), api.dirichlets.cpu())
    assert torch.equal(dev.pi_hat.cpu(), api.pi_hat.cpu())
    assert torch.equal(dev.get_pbest().cpu(), api.get_pbest().cpu())
    assert dev.labeled_idxs == api.labeled_idxs and dev.labels == api.labels


def _assert_history(dev, exp, n0=0):
    idx, q, tie = dev.history()
    best, best_tie = dev.best_history()
    e_idx, e_q, e_tie, e_best = exp
    assert idx[n0:].tolist() == e_idx
    assert q[n0:].tobytes() == np.asarray(e_q, np.float32).tobytes()
    assert tie[n0:].tolist() == e_tie
    assert best[n0:].tolist() == e_best and not best_tie.any()


def _parity(kind, k, shards=None, data=None, kw=None, until_tie=False):
    """``until_tie``: where the API path breaks an isclose tie with random.choice (EIG / entropy ties), the loop takes
    the first maximum and flags the step (DESIGN.md §6 (xi)): compare up to that step, which must be flagged."""
    preds, labels = data or _data()
    kw = kw or KINDS[kind]
    random.seed(3)
    api = _make(preds, labels, kw, shards)
    exp = _api_steps(api, labels, k)
    st_api = random.getstate()
    random.seed(3)
    dev = _make(preds, labels, kw, shards)
    dev.run_steps(k, labels, record_best=True)
    if until_tie and 1 in exp[2]:
        t = exp[2].index(1)
        idx, _q, tie = dev.history()
        assert idx[:t].tolist() == exp[0][:t] and tie[:t + 1].tolist() == exp[2][:t + 1]
        return dev, exp
    assert random.getstate() == st_api
    _assert_history(dev, exp)
    _assert_same_state(dev, api)
    return dev, exp


@pytest.mark.parametrize("graph", ["1", "0"])
@pytest.mark.parametrize("shards", [1, 2, 3])
@pytest.mark.parametrize("kind", list(KINDS))
def test_device_loop_equals_the_api_loop(kind, shards, graph, monkeypatch):
    monkeypatch.setenv("CODA_B200_GRAPH", graph)
    dev, exp = _parity(kind, 12, shards)
    # iid: n_s > 1 every step; prefilter: every step sampled; uncertainty: no draw without a tie
    assert dev.stochastic == (kind != "uncertainty")
    if kind == "iid":
        assert exp[2] == [1] * 12                           # flagged: the reference drew with random.choice


def _golden():
    with open(f"{GOLDEN}/acquisitions.json") as f:
        return json.load(f)


def _rng_digest():
    import hashlib
    return hashlib.sha256(repr(random.getstate()).encode()).hexdigest()[:16]


@pytest.mark.parametrize("kind", ["iid", "uncertainty", "prefilter"])
def test_device_loop_reproduces_the_reference_goldens(kind):
    from coda_b200 import CODA, TensorDataset
    from coda_b200.synth import synth
    g = _golden()[kind]
    preds, labels = synth(g["H"], g["N"], g["C"], seed=g["data_seed"])
    kw = dict(prefilter_n=g["prefilter_n"]) if kind == "prefilter" else dict(q=kind)
    random.seed(g["seed"])
    sel = CODA(TensorDataset(preds.cuda(), labels.cuda()), **kw)
    k = len(g["steps"])
    sel.run_steps(k, labels, record_best=True)
    idx, q, _tie = sel.history()
    best, _ = sel.best_history()
    assert idx.tolist() == [s["idx"] for s in g["steps"]]
    # uncertainty: the entropy of the slab scan's ensemble sums, as on the API path, is within an ulp of the reference's
    assert np.abs(q.astype(np.float64) - [s["q"] for s in g["steps"]]).max() < (2e-6 if kind == "prefilter" else 3e-7)
    assert _rng_digest() == g["steps"][-1]["rng"]
    if "best" in g["steps"][0]:
        assert best.tolist() == [s["best"] for s in g["steps"]]
    if kind == "prefilter":
        assert sel.stochastic and g["stochastic"]


def _candidate_counts(sel):
    d = u = 0
    for e in sel.engines:
        dd, uu = e.candidate_counts()
        d, u = d + dd, u + uu
    return d, u


@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("kind", ["iid", "uncertainty", "prefilter"])
def test_runs_across_the_sample_size_and_the_all_unlabeled_fallback(kind, shards, monkeypatch):
    """A run long enough that the disagreeing candidates run out (coda.py:239 fallback); for the prefilter it first
    crosses n_s <= prefilter_n (plain arg-max), with pre-draws spread over several chunks."""
    from coda_b200 import selector
    data = _data(N=300, disagree=24)
    kw = dict(prefilter_n=5) if kind == "prefilter" else KINDS[kind]
    monkeypatch.setattr(selector, "ABL_CHUNK_WORDS", 3 * 6)     # 3 prefilter rows / 9 iid rows per chunk
    probe = _make(*data, kw, shards)
    d0, u0 = _candidate_counts(probe)
    probe.close()
    assert 10 < d0 <= 24 and u0 == 300
    _parity(kind, d0 + 4, shards, data=data, kw=kw, until_tie=kind != "iid")


def test_predicted_candidate_counts_hold_on_the_device():
    from coda_b200.selector import candidate_counts
    preds, labels = _data(N=300, disagree=24)
    sel = _make(preds, labels, dict(q="iid"))
    d0, u0 = _candidate_counts(sel)
    pred = candidate_counts(d0, u0, d0 + 3)
    for s in range(d0 + 3):
        d, u = _candidate_counts(sel)
        assert (d if d > 0 else u) == pred[s]
        sel.run_steps(1, labels)
    sel.history()


def _dup_columns(N=400, copies=3):
    """Items n and n + N/copies... hold the same predictions: equal entropies and EIGs, exact ties."""
    base, labels = _data(N=N // copies, seed=5)
    preds = base.repeat(1, copies, 1)
    return preds, labels.repeat(copies)


@pytest.mark.parametrize("kind", ["uncertainty", "prefilter"])
def test_exact_ties_take_the_first_and_are_flagged(kind):
    preds, labels = _dup_columns()
    if kind == "prefilter":
        # a sample of all candidates but one holds at least two of the three copies of the best item
        probe = _make(preds, labels, dict(q="iid"))
        m = _candidate_counts(probe)[0] - 1
        probe.close()
        kw = dict(prefilter_n=m)
    else:
        kw = dict(q="uncertainty")
    random.seed(1)
    sel = _make(preds, labels, kw)
    if kind == "uncertainty":
        from coda_b200.baselines import ensemble_entropy
        qv = ensemble_entropy(sel._cat("ens"), sel.H).cpu()
        mask = sel._candidate_mask(sel._cat("labeled"), sel._cat("disagree")).cpu()
        first = int(torch.nonzero(qv == qv[mask].max())[0, 0])
        sel.run_steps(1, labels)
        idx, q, tie = sel.history()
        assert idx.tolist() == [first] and tie.tolist() == [1] and q[0] == np.float32(qv[first])
        return
    # prefilter: the first sampled position among the exact maxima of the sample
    sel._fetch_report()                                     # the scoring pass (no random draws)
    state = random.getstate()
    d0, _u0 = _candidate_counts(sel)
    ids = torch.nonzero((sel._cat("labeled") == 0) & (sel._cat("disagree") != 0)).flatten().tolist()
    pos = random.sample(range(d0), m)
    eig = sel.eig.cpu()
    qv = eig[[ids[p] for p in pos]]
    random.setstate(state)
    sel.run_steps(1, labels)
    idx, q, tie = sel.history()
    loc = int(torch.nonzero(qv == qv.max())[0, 0])
    assert idx.tolist() == [ids[pos[loc]]] and q[0] == qv[loc].item()
    assert int((qv == qv.max()).sum()) >= 2 and tie.tolist() == [1]


@pytest.mark.parametrize("kind", list(KINDS))
def test_api_and_device_steps_interleave(kind):
    preds, labels = _data()
    kw = KINDS[kind]
    random.seed(9)
    api = _make(preds, labels, kw)
    exp = _api_steps(api, labels, 9)
    st_api = random.getstate()
    random.seed(9)
    mix = _make(preds, labels, kw, shards=2)
    a = _api_steps(mix, labels, 2)
    mix.run_steps(5, labels, record_best=True)
    b = _api_steps(mix, labels, 2)
    assert random.getstate() == st_api
    idx, q, tie = mix.history()                             # the five device-loop steps
    assert idx.tolist() == exp[0][2:7]
    assert q.tobytes() == np.asarray(exp[1][2:7], np.float32).tobytes()
    assert tie.tolist() == exp[2][2:7]
    assert mix.best_history()[0].tolist() == exp[3][2:7]
    assert a[0] + b[0] == exp[0][:2] + exp[0][7:] and a[3] + b[3] == exp[3][:2] + exp[3][7:]
    _assert_same_state(mix, api)


@pytest.mark.parametrize("fmt", ["fp16", "compact"])
@pytest.mark.parametrize("kind", ["iid", "uncertainty"])
def test_slab_formats(kind, fmt):
    from coda_b200 import CODA, CompactDataset, TensorDataset
    if fmt == "fp16":
        preds, labels = _data()
        make = lambda: CODA(TensorDataset(preds.half().cuda(), labels.cuda()), q=kind)      # noqa: E731
    else:
        from coda_b200 import CompactSlab
        from coda_b200.synth import synth_compact
        ids, probs, labels = synth_compact(12, 700, 20, 3, seed=4)
        slab = CompactSlab(ids, probs, 20).to("cuda:0")
        make = lambda: CODA(CompactDataset(slab, labels.cuda()), q=kind)                   # noqa: E731
    random.seed(2)
    api = make()
    exp = _api_steps(api, labels, 10)
    st = random.getstate()
    random.seed(2)
    dev = make()
    dev.run_steps(10, labels, record_best=True)
    assert random.getstate() == st
    _assert_history(dev, exp)
    _assert_same_state(dev, api)


def _refused(sel, labels, exc, match):
    state = random.getstate()
    d = sel.dirichlets.clone()
    ctr = int(sel.engine.step_ctr.item())
    launches = sel.engine.counters["launches"]
    with pytest.raises(exc, match=match):
        sel.run_steps(3, labels)
    assert random.getstate() == state and sel.engine.counters["launches"] == launches
    assert int(sel.engine.step_ctr.item()) == ctr and torch.equal(sel.dirichlets, d) and not sel.labeled_idxs


def test_refusals_raise_before_any_launch(monkeypatch):
    preds, labels = _data(N=200)
    random.seed(0)
    _refused(_make(preds, labels, dict(q="iid", prefilter_n=5)), labels, NotImplementedError, "prefilter_n")
    _refused(_make(preds, labels, dict(q="uncertainty", prefilter_n=5)), labels, NotImplementedError, "prefilter_n")
    _refused(_make(preds, labels, dict(q="margin")), labels, NotImplementedError, "margin")
    for kw in (dict(q="iid"), dict(q="uncertainty"), dict(prefilter_n=5)):
        sel = _make(preds, labels, kw)
        sel.group = types.SimpleNamespace(world=2)          # as built by one process per GPU (this process: one shard)
        _refused(sel, labels, NotImplementedError, "one process per GPU")
    monkeypatch.setenv("CODA_B200_ENS", "0")
    _refused(_make(preds, labels, dict(q="uncertainty")), labels, RuntimeError, "ensemble sums")
