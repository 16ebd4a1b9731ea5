"""Scoring only the prefilter_n sample (csrc/sample.cu) on the GPU: every scored item's EIG is the bits the full
incremental pass gives it, so the sample path and the full path (forced with CODA_B200_PREFILTER_SCORING) make the
same picks, q values, tie flags, posterior and Python random state, on the API path and in run_steps."""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _data(H, N, C, seed=11, disagree=None):
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, seed=seed)
    if disagree is not None:       # only the first `disagree` items can have disagreeing models
        rest = preds[:, disagree:]
        onehot = torch.nn.functional.one_hot(rest[0].argmax(-1), C).to(preds.dtype)
        preds[:, disagree:] = 0.5 * rest + 0.5 * onehot
    return preds, labels


def _make(preds, labels, scoring, monkeypatch, shards=None, **kw):
    from coda_b200 import CODA, TensorDataset
    monkeypatch.setenv("CODA_B200_PREFILTER_SCORING", scoring)
    return CODA(TensorDataset(preds.to("cuda"), labels.cuda()), shards=shards, **kw)


@pytest.mark.parametrize("shape", [(10, 600, 6), (48, 20000, 20), (256, 1500, 100), (300, 800, 12), (33, 1507, 12)])
@pytest.mark.parametrize("m", [1, 7, 50, "all"])
def test_sampled_eig_is_the_full_pass_bits(shape, m, monkeypatch):
    """Teacher-forced: A scores only its sample, B (no prefilter) scores every item; at every step A's EIG at the items
    it scored equals B's bit for bit."""
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    preds, labels = _data(*shape)
    d0 = int(_make(preds, labels, "full", monkeypatch).engine.candidate_counts()[0])
    mm = d0 + 5 if m == "all" else m
    random.seed(1)
    a = _make(preds, labels, "sample", monkeypatch, prefilter_n=mm)
    b = _make(preds, labels, "auto", monkeypatch)
    assert a.engine.sample_scoring and not b.engine.sample_scoring
    assert a.engine.use_tc == (shape[0] <= 256)
    for _ in range(4):
        idx, q = a.get_next_item_to_label()
        items = a.engine.sw["items"]
        items = items[items >= 0].long()
        assert items.numel() == min(mm, d0)
        b.get_next_item_to_label()
        assert torch.equal(a.eig[items], b.eig[items])
        assert q == float(b.eig[idx])
        for s in (a, b):
            s.add_label(idx, int(labels[idx]), q)
        d0 -= 1


def _api(sel, labels, k):
    out = []
    for _ in range(k):
        i, q = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), q)
        out.append((int(i), np.float32(q).tobytes(), int(sel.get_best_model_prediction())))
    return out


def _state(sel):
    return (sel.stochastic, sel.dirichlets.cpu(), sel.pi_hat.cpu(), sel.get_pbest().cpu(), sel.pi_hat_xi.cpu(),
            list(sel.labeled_idxs))


def _same_state(x, y):
    assert x[0] == y[0] and x[5] == y[5]
    for u, v in zip(x[1:5], y[1:5]):
        assert torch.equal(u, v)


def _run(preds, labels, scoring, monkeypatch, how, k, shards=None, rule="first", **kw):
    random.seed(7)
    sel = _make(preds, labels, scoring, monkeypatch, shards=shards, **kw)
    assert sel.engine.sample_scoring == (scoring == "sample")
    if how == "api":
        out = _api(sel, labels, k)
    else:
        sel.run_steps(k, labels.cuda(), record_best=True, tie_rule=rule)
        idx, q, tie = sel.history()
        best, _ = sel.best_history()
        out = (idx.tolist(), q.tobytes(), tie.tolist(), best.tolist())
    st = _state(sel)
    rs = random.getstate()
    sel.close()
    return out, st, rs


@pytest.mark.parametrize("graph", ["1", "0"])
@pytest.mark.parametrize("shards", [1, 2, 3])
@pytest.mark.parametrize("how,rule", [("api", "first"), ("loop", "first"), ("loop", "reference")])
def test_sample_path_equals_full_path(how, rule, shards, graph, monkeypatch):
    monkeypatch.setenv("CODA_B200_GRAPH", graph)
    preds, labels = _data(12, 1200, 6, seed=17)
    got = [_run(preds, labels, sc, monkeypatch, how, 10, shards, rule, prefilter_n=40) for sc in ("sample", "full")]
    (o1, s1, r1), (o2, s2, r2) = got
    assert o1 == o2 and r1 == r2
    _same_state(s1, s2)


@pytest.mark.parametrize("env", [dict(CODA_B200_TC="0"), dict(dtype="f16"), dict(compact="1")])
def test_sample_path_on_other_slabs_and_row_kernels(env, monkeypatch):
    from coda_b200.synth import synth_compact
    preds, labels = _data(40, 1500, 100, seed=3)
    if env.get("CODA_B200_TC"):
        monkeypatch.setenv("CODA_B200_TC", env["CODA_B200_TC"])
    if env.get("dtype"):
        preds = preds.half()
    kw = dict(prefilter_n=30)
    if env.get("compact"):
        from coda_b200 import CompactSlab
        ids, probs, labels = synth_compact(40, 1500, 100, K=4, seed=3)
        preds = CompactSlab(ids, probs, 100)
    for how in ("api", "loop"):
        got = [_run(preds, labels, sc, monkeypatch, how, 8, **kw) for sc in ("sample", "full")]
        assert got[0][0] == got[1][0] and got[0][2] == got[1][2]
        _same_state(got[0][1], got[1][1])


@pytest.mark.parametrize("shards", [1, 2])
@pytest.mark.parametrize("how,rule", [("api", "first"), ("loop", "first"), ("loop", "reference")])
def test_phase_boundaries(how, rule, shards, monkeypatch):
    """Sampled steps, then n_s <= prefilter_n (the identity sample: every candidate, no random draw), then the
    all-unlabeled fallback (more candidates than the sample holds: every item scored in chunks), pre-draws over
    chunks.  The full path runs the EIG loop for the last two phases."""
    from coda_b200 import selector
    monkeypatch.setattr(selector, "ABL_CHUNK_WORDS", 3 * 6)
    preds, labels = _data(12, 600, 6, seed=17, disagree=14)
    got = [_run(preds, labels, sc, monkeypatch, how, 24, shards, rule, prefilter_n=5) for sc in ("sample", "full")]
    assert got[0][0] == got[1][0] and got[0][2] == got[1][2]
    _same_state(got[0][1], got[1][1])


@pytest.mark.parametrize("tc", ["1", "0"])
def test_scratch_rows_equal_the_cached_rows(tc, monkeypatch):
    """Teacher-forced: the scratch rows of A's sample equal the cached rows of B (full scoring) for the same
    (item, class), and A's cached template rows equal B's."""
    monkeypatch.setenv("CODA_B200_TC", tc)
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    preds, labels = _data(40, 3000, 10, seed=5)
    random.seed(2)
    sel = _make(preds, labels, "sample", monkeypatch, prefilter_n=64)
    full = _make(preds, labels, "auto", monkeypatch)
    e, f = sel.engine, full.engine
    assert e.use_tc == (tc == "1")
    for _ in range(3):
        idx, q = sel.get_next_item_to_label()
        full.get_next_item_to_label()
        for s in (sel, full):
            s.add_label(idx, int(labels[idx]), q)
    e.sw["rows"].fill_(float("nan"))
    sel.get_next_item_to_label()
    full.get_next_item_to_label()
    e.sync()
    f.sync()
    assert torch.equal(e.ph_cache, f.ph_cache[: e.T])
    items, hoff = e.sw["items"].cpu(), e.sw["hoff"].cpu()
    heavy_off = e.heavy_off.cpu()
    n_rows = 0
    for j, n in enumerate(items.tolist()):
        if n < 0:
            continue
        k = int(heavy_off[n + 1] - heavy_off[n])
        got = e.sw["rows"][int(hoff[j]): int(hoff[j]) + k]
        ref = f.ph_cache[e.T + int(heavy_off[n]): e.T + int(heavy_off[n]) + k]
        assert torch.equal(got, ref)
        n_rows += k
    assert n_rows == int(e.sw["nheavy"]) > 0


def test_choice_knob_and_refusals(monkeypatch):
    from coda_b200 import engine as eng
    preds, labels = _data(10, 800, 6)
    r = eng.PREFILTER_ROW_COST_RATIO
    m_lo = int(800 / r)
    assert _make(preds, labels, "auto", monkeypatch, prefilter_n=m_lo).engine.sample_scoring
    assert not _make(preds, labels, "auto", monkeypatch, prefilter_n=m_lo + 1).engine.sample_scoring
    assert not _make(preds, labels, "auto", monkeypatch, prefilter_n=m_lo, q="iid").engine.sample_scoring
    assert not _make(preds, labels, "auto", monkeypatch, prefilter_n=m_lo, mode="recompute").engine.sample_scoring
    assert _make(preds, labels, "sample", monkeypatch, prefilter_n=700).engine.sample_scoring
    assert not _make(preds, labels, "full", monkeypatch, prefilter_n=5).engine.sample_scoring
    with pytest.raises(ValueError, match="PREFILTER_SCORING"):
        _make(preds, labels, "always", monkeypatch, prefilter_n=5)
    with pytest.raises(ValueError, match="incremental"):
        _make(preds, labels, "sample", monkeypatch, prefilter_n=5, mode="recompute")
    e = _make(preds, labels, "sample", monkeypatch, prefilter_n=50).engine
    heavy = (e.heavy_off[1:] - e.heavy_off[:-1]).cpu()
    assert e.n_heavy > 0
    # T template rows + the scratch, no heavy-row cache
    assert e.ph_cache.shape == (e.T, e.Hp) and e.gain is None
    assert e.sw["cap"] == max(1, int(heavy.topk(50).values.sum()))
    assert e.sw["rows"].shape == (e.sw["cap"], e.Hp)
    assert int(e.tiles[:, 2].sum()) == e.T                 # the tile lists cover the template positions only
    with pytest.raises(RuntimeError, match="prefilter samples"):
        with e._on():
            e.scored = False
            e._score()
    f = _make(preds, labels, "full", monkeypatch, prefilter_n=50).engine
    assert f.ph_cache.shape == (f.npairs, f.Hp) and f.sw is None
