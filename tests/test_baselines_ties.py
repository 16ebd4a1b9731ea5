"""The competing selectors' ``run_steps(..., tie_rule="reference")`` on the GPU: the draws the reference makes from
torch's CPU and CUDA generators, made from device replicas of them (csrc/bl_ref.cu), against the reference goldens,
against the API path call for call (picks, best models, sums, and every generator's state byte for byte), across
layouts, on tie-heavy tasks, and the replicas on their own against torch."""
import random

import numpy as np
import pytest
import torch

from test_baselines_loop import _cases, _golden_selector, _load, _make, _py_digest, _seed_all
from test_baselines_ties_host import TorchCpuModel, cuda_randint

pytestmark = pytest.mark.gpu

METHODS = ["iid", "uncertainty", "activetesting", "vma", "model_picker"]


def _torch_digest():
    import hashlib
    return int.from_bytes(hashlib.sha256(torch.get_rng_state().numpy().tobytes()).digest()[:8], "little", signed=True)


def _rng_states():
    return random.getstate(), torch.get_rng_state(), torch.cuda.get_rng_state(torch.device("cuda:0"))


def _same_rng(a, b):
    return a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


# -- against the reference goldens ----------------------------------------------------------------------------------
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("method", ["iid", "activetesting", "vma"])
def test_reference_rule_reproduces_the_goldens_at_every_step(method, split):
    """Picks, q and the best model of every step are the reference's, ties included, and torch's CPU generator ends
    (and, split, stands after every call) where the reference's does."""
    for name in _cases(method):
        g = _load(name)
        sel, labels = _golden_selector(g, method)
        assert int(sel.get_best_model_prediction()) == int(g["best0"])
        steps = int(g["steps"])
        parts = [1, 7, steps - 8] if split else [steps]
        done = 0
        for k in parts:
            assert sel.run_steps(k, labels, tie_rule="reference") == k
            done += k
            assert _torch_digest() == int(g["torch"][done - 1]), (name, done)
            assert _py_digest() == int(g["py"][done - 1]), (name, done)
        idx, q, tie = sel.history()
        best, _btie = sel.best_history()
        assert idx.tolist() == g["idx"].tolist(), name
        np.testing.assert_allclose(q, g["q"], rtol=1e-5)
        assert best.tolist() == g["best"].tolist(), name
        assert sel.d_l_idxs == g["idx"].tolist()
        sel.close()


def _ill_conditioned(g, method, s, labeled):
    """More than one unlabeled item is within fp32 noise of the reference's best score at step s."""
    if method == "model_picker":
        from test_baselines import _ref_tol
        ref = g["ent"][s]
        m = np.nanmin(ref)
        return int(np.sum(ref <= m + _ref_tol(int(g["C"]), ref))) > 1
    score = g["score"].copy()
    score[np.asarray(labeled, np.int64)] = -np.inf
    top2 = np.sort(score)[-2:]
    return top2[1] - top2[0] <= 1e-6


@pytest.mark.parametrize("method", ["uncertainty", "model_picker"])
def test_reference_rule_follows_the_goldens_while_the_picks_agree(method):
    """Uncertainty and ModelPicker, one call per step: while the picks are the reference's, so are torch's CPU state
    after the step and (Uncertainty) the best model.  The ModelPicker goldens hold the CPU stream only (their best model
    was drawn on the CPU): its CUDA draws are checked against the API path below."""
    for name in _cases(method):
        g = _load(name)
        sel, labels = _golden_selector(g, method)
        sel.get_best_model_prediction()
        agreed = 0
        for s in range(int(g["steps"])):
            sel.run_steps(1, labels, tie_rule="reference")
            idx, _q, _tie = sel.history()
            if int(idx[s]) != int(g["idx"][s]):            # only where the reference's own scores are within fp32 noise
                assert _ill_conditioned(g, method, s, labeled=idx[:s]), (name, s)
                break
            assert _torch_digest() == int(g["torch"][s]), (name, s)
            assert _py_digest() == int(g["py"][s]), (name, s)
            if method == "uncertainty":
                assert int(sel.best_history()[0][s]) == int(g["best"][s]), (name, s)
            agreed += 1
        assert agreed >= 2, name
        sel.close()


# -- against the API path -------------------------------------------------------------------------------------------
def _drive(method, preds, labels, plan, **kw):
    """Run ``plan`` [("api" | "dev", steps)] from the goldens' seeding -> (picks, q, best per step, the selector's
    sums, tie flags of the device steps, the generators' states)."""
    _seed_all()
    sel = _make(method, preds, labels.cuda(), **kw)
    qs, bests = [], []
    seen = 0
    for kind, n in plan:
        if kind == "api":
            for _ in range(n):
                i, q = sel.get_next_item_to_label()
                sel.add_label(i, int(labels[i]), q)
                qs.append(float(q))
                bests.append(int(sel.get_best_model_prediction()))
        else:
            assert sel.run_steps(n, labels, tie_rule="reference") == n
            _idx, q, _tie = sel.history()
            best, _bt = sel.best_history()
            qs += q[seen:].tolist()
            bests += best[seen:].tolist()
            handed = n - (len(q) - seen)                  # steps the API path finished after a stop (not in history)
            qs += [None] * handed
            bests += [None] * handed
            seen = len(q)
    rng = _rng_states()
    sums = {}
    if method in ("iid", "uncertainty"):
        sums["risk"] = sel._risk_sum.cpu().numpy()
    elif method == "model_picker":
        sums["counts"] = sel.correct_counts.cpu().numpy()
        sums["post"] = sel.posterior.cpu().numpy()
        sums["n_disagree"] = sel._n_disagree
    else:
        sums["lure"] = sel.get_risk_estimates().cpu().numpy()
        sums["qs"] = list(sel.qs)
    ties = [a.tolist() for a in (sel.history()[2], sel.best_history()[1])]
    out = dict(picks=list(sel.d_l_idxs), q=qs, best=bests, sums=sums, ties=ties, rng=rng,
               stochastic=bool(sel.stochastic))
    sel.close()
    return out


def _assert_same_run(got, want, tag):
    assert got["picks"] == want["picks"], tag
    for key in ("q", "best"):
        assert [w if g is None else g for g, w in zip(got[key], want[key])] == want[key], (tag, key)
    for key, v in want["sums"].items():
        if key == "post":                              # the device sums the posterior in fp64 (DESIGN.md §6)
            np.testing.assert_allclose(got["sums"][key], v, rtol=1e-6, atol=0, err_msg=tag)
        elif key == "lure":
            np.testing.assert_allclose(got["sums"][key], v, rtol=1e-6, atol=1e-7, err_msg=tag)
        else:
            assert np.array_equal(np.asarray(got["sums"][key]), np.asarray(v)), (tag, key)
    assert got["stochastic"] == want["stochastic"], tag
    assert _same_rng(got["rng"], want["rng"]), tag


def _tie_task():
    """Duplicated models (the best model ties with its copy) and duplicated items (Uncertainty's and ModelPicker's
    picks tie with their twins)."""
    from coda_b200.synth import synth
    preds, labels = synth(24, 200, 10, 11)
    preds = torch.cat([preds, preds[:8]], 0)
    preds = torch.cat([preds, preds], 1).contiguous()
    return preds, torch.cat([labels, labels])


PLAN = [("api", 3), ("dev", 10), ("api", 2), ("dev", 12)]


@pytest.mark.parametrize("method", METHODS)
def test_reference_rule_equals_the_api_path_across_layouts(method, monkeypatch):
    from coda_b200 import CompactSlab
    from coda_b200.synth import synth_compact
    preds, labels = _tie_task()
    steps = sum(n for _, n in PLAN)
    want = _drive(method, preds.cuda(), labels, [("api", steps)])
    runs = {}
    for tag, kw, env in (("1", {}, "1"), ("2", {"shards": 2}, "1"), ("3", {"shards": 3}, "1"), ("eager", {}, "0")):
        monkeypatch.setenv("CODA_B200_GRAPH", env)
        runs[tag] = _drive(method, preds.cuda(), labels, PLAN, **kw)
        _assert_same_run(runs[tag], want, tag)
    for tag in ("2", "3", "eager"):
        assert runs[tag]["ties"] == runs["1"]["ties"], tag
    assert any(runs["1"]["ties"][1]), "the task has no best-model tie"
    monkeypatch.setenv("CODA_B200_GRAPH", "1")
    half = preds.half()
    _assert_same_run(_drive(method, half.cuda(), labels, PLAN), _drive(method, half.cuda(), labels, [("api", steps)]),
                     "f16")
    ids, probs, clabels = synth_compact(16, 300, 20, 4, seed=5)
    cs = CompactSlab(ids, probs, 20).to(torch.device("cuda:0"))
    _assert_same_run(_drive(method, cs, clabels, PLAN, shards=2), _drive(method, cs, clabels, [("api", steps)]),
                     "compact")


@pytest.mark.parametrize("method", METHODS)
def test_reference_rule_with_one_model(method):
    from coda_b200.synth import synth
    preds, labels = synth(1, 300, 5, 3)
    _assert_same_run(_drive(method, preds.cuda(), labels, [("dev", 8), ("api", 2), ("dev", 10)]),
                     _drive(method, preds.cuda(), labels, [("api", 20)]), "H=1")


def test_uncertainty_ties_over_thousands_of_items():
    """Every item the same: each step ties among all unlabeled items, so randperm's skip crosses several twists."""
    H, N, C = 4, 2600, 3
    preds = torch.full((H, N, C), 0.25)
    preds[:, :, 0] = 0.5
    labels = torch.zeros(N, dtype=torch.int64)
    got = _drive("uncertainty", preds.cuda(), labels, [("dev", 12), ("api", 1), ("dev", 6)])
    want = _drive("uncertainty", preds.cuda(), labels, [("api", 19)])
    _assert_same_run(got, want, "all tied")
    assert all(got["ties"][0])


@pytest.mark.parametrize("method", ["iid", "uncertainty", "model_picker"])
def test_chunked_runs_past_the_history_ring(method, monkeypatch):
    import coda_b200.baselines as bl
    monkeypatch.setattr(bl, "HIST_CAP", 8)
    preds, labels = _tie_task()
    _assert_same_run(_drive(method, preds.cuda(), labels, [("dev", 30)]),
                     _drive(method, preds.cuda(), labels, [("api", 30)]), "HIST_CAP 8")


def test_vma_hand_over_continues_from_the_replicas():
    """VMA's weights vanish after j labels; the API path finishes the run from torch's state as the replica left it."""
    H, N, C, j = 8, 120, 4, 6
    g = torch.Generator().manual_seed(0)
    preds = torch.full((H, N, C), 0.1)
    preds[:, :, 0] = 0.7
    for n in range(j):
        preds[H - 2:, n, 0] = 0.1
        preds[H - 2:, n, 1] = 0.7
    labels = torch.randint(0, C, (N,), generator=g)
    want = _drive("vma", preds.cuda(), labels, [("api", 15)])
    _seed_all()
    sel = _make("vma", preds.cuda(), labels.cuda())
    assert sel.run_steps(15, labels, tie_rule="reference") == 15
    assert len(sel.history()[0]) == j
    assert sel.d_l_idxs == want["picks"]
    assert _same_rng(_rng_states(), want["rng"])
    sel.close()


def test_switching_rules_recaptures_the_step(monkeypatch):
    """Reference, default and reference steps in turn on one selector: each rule replays its own graph, so the run
    equals the same calls with the kernels launched one by one."""
    preds, labels = _tie_task()
    out = []
    for env in ("1", "0"):
        monkeypatch.setenv("CODA_B200_GRAPH", env)
        _seed_all()
        sel = _make("uncertainty", preds.cuda(), labels.cuda())
        sel.run_steps(5, labels, tie_rule="reference")
        sel.run_steps(10, labels, seed=3)
        sel.run_steps(5, labels, tie_rule="reference")
        out.append(([a.tolist() for a in sel.history() + sel.best_history()], _rng_states()))
        sel.close()
    assert out[0][0] == out[1][0]
    assert _same_rng(out[0][1], out[1][1])


# -- the replicas on their own --------------------------------------------------------------------------------------
def _rng_run(ops, trng, grng):
    from coda_b200 import _native as nat
    dev = trng.device
    ops_t = torch.tensor(ops, dtype=torch.int64, device=dev)
    out = torch.empty(len(ops), dtype=torch.int64, device=dev)
    nat.call("coda_b200_torch_rng_run", trng.data_ptr(), grng.data_ptr(), ops_t.data_ptr(), len(ops), out.data_ptr(),
             torch.cuda.current_stream(dev).cuda_stream)
    return out.tolist()


@pytest.mark.parametrize("seed", [0, 12345, (1 << 63) + 5])
def test_cuda_replica_is_torch_randint_on_the_device(seed):
    from coda_b200.baselines import cuda_rng_state, cuda_rng_words, torch_rng_words
    dev = torch.device("cuda:0")
    torch.cuda.manual_seed(seed)
    torch.rand(5000, device=dev)                         # an offset that is not a multiple of one call's
    st = torch.cuda.get_rng_state(dev)
    grng = cuda_rng_words(st).to(dev)
    trng = torch_rng_words(torch.get_rng_state()).to(dev)
    ns = [1, 2, 3, 7, 24, 1000, 1024, 65_537, (1 << 28) - 1] * 3
    got = _rng_run([[2, n] for n in ns], trng, grng)
    off = int(cuda_rng_words(st)[1])
    assert got[0] == cuda_randint(seed, off, ns[0]) and got[1] == cuda_randint(seed, off + 4, ns[1])
    want = [int(torch.randint(n, (1,), device=dev)) for n in ns]
    assert got == want
    assert torch.equal(cuda_rng_state(grng.cpu()), torch.cuda.get_rng_state(dev))


def test_cpu_replica_is_torch_on_the_host():
    from coda_b200.baselines import cuda_rng_words, torch_rng_state, torch_rng_words
    dev = torch.device("cuda:0")
    torch.manual_seed(4)
    st = torch.get_rng_state()
    trng = torch_rng_words(st).to(dev)
    grng = cuda_rng_words(torch.cuda.get_rng_state(dev)).to(dev)
    ops = [[0, 2], [1, 1], [0, 2500], [1, 7], [1, (1 << 28) + 3], [0, 624], [1, 1 << 40], [0, 1], [0, 70_000],
           [1, 1000]]
    got = _rng_run(ops, trng, grng)
    model = TorchCpuModel(st)
    assert got == [model.randperm0(n) if k == 0 else model.randint(n) for k, n in ops]
    want = [int(torch.randperm(n)[0]) if k == 0 else int(torch.randint(n, (1,))[0]) for k, n in ops]
    assert got == want
    assert torch.equal(torch_rng_state(trng.cpu(), st), torch.get_rng_state())
