"""ModelPicker's epsilon grid search on the GPU (coda_b200.eps_search, csrc/eps_search.cu): every sampled run (e, r) is
bit for bit ModelPicker.run_steps on that run's pool, the picks follow a NumPy restatement of modelpicker.py while it
is well conditioned, and the labels, pool accuracies and metrics equal exact host computations."""
import numpy as np
import pytest
import torch

from test_baselines import _fp64_entropies, _ref_tol

pytestmark = pytest.mark.gpu

SCRIPT_EPS = (0.35, 0.36, 0.37, 0.38, 0.39, 0.40, 0.41, 0.42, 0.43, 0.44, 0.45, 0.46, 0.47, 0.48, 0.49)


def _hard(preds):
    """[N][H] int64 hard predictions of a dense (H, N, C) slab."""
    return preds.float().argmax(2).t().cpu().numpy().astype(np.int64)


def _majority(hard):
    out = np.zeros(hard.shape[0], dtype=np.int64)
    for i, row in enumerate(hard):
        vals, cnts = np.unique(row, return_counts=True)
        out[i] = vals[np.argmax(cnts)]
    return out


def _subset(preds, pool):
    from coda_b200 import CompactSlab
    idx = torch.as_tensor(pool, device=preds.device)
    if isinstance(preds, CompactSlab):
        return CompactSlab(preds.ids[:, idx].contiguous(), preds.probs[:, idx].contiguous(), preds.shape[2])
    return preds[:, idx].contiguous()


def _check_contract(preds, res, runs):
    """Run (e, r) against ModelPicker.run_steps on pool r with the run's key: picks, best models and tie flags."""
    from coda_b200 import ModelPicker, TensorDataset
    from coda_b200.eps_search import eps_search_run_key
    from coda_b200.datasets import CompactDataset, CompactSlab
    B = res["picks"].shape[2]
    for e, r in runs:
        pool = res["realisations"][r]
        sub = _subset(preds, pool)
        ds = CompactDataset(sub) if isinstance(sub, CompactSlab) else TensorDataset(sub)
        sel = ModelPicker(ds, epsilon=res["epsilons"][e])
        lab = torch.as_tensor(res["labels"][pool], dtype=torch.int64, device="cuda")
        sel.run_steps(B, lab, seed=eps_search_run_key(res["seed"], e, r))
        idx, _q, tie = sel.history()
        best, btie = sel.best_history()
        sel.close()
        assert np.array_equal(idx, res["picks"][e, r]), (e, r)
        assert np.array_equal(tie, res["pick_tie"][e, r]), (e, r)
        assert np.array_equal(best, res["best"][e, r]), (e, r)
        assert np.array_equal(btie, res["best_tie"][e, r]), (e, r)


def _sample(E, R, k=4, rng=None):
    rng = rng or np.random.default_rng(0)
    runs = {(0, 0), (E - 1, R - 1)}
    while len(runs) < min(k, E * R):
        runs.add((int(rng.integers(E)), int(rng.integers(R))))
    return sorted(runs)


@pytest.mark.parametrize("H,C", [(1, 2), (5, 10), (32, 100), (33, 10), (256, 100), (1024, 2), (1024, 100)])
def test_runs_equal_run_steps_bit_for_bit(H, C):
    from coda_b200 import TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth
    N = 400 if H < 1024 else 160
    preds, _ = synth(H, N, C, seed=H + C)
    preds = preds.cuda()
    np.random.seed(H)
    eps = SCRIPT_EPS if H >= 256 else (0.3, 0.46, 0.5, 0.7)
    res = modelpicker_eps_search(TensorDataset(preds), epsilons=eps, iterations=5, pool_size=60, budget=40,
                                 seed=1000 + H)
    assert res["picks"].shape == (len(eps), 5, 40)
    _check_contract(preds, res, _sample(len(eps), 5))


def test_unanimous_and_duplicated_items_and_models_through_the_last_label():
    """budget = pool size crosses n_disagree = 0; duplicated models and items give exact ties in both draws."""
    from coda_b200 import TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth
    H, N, C = 12, 120, 6
    preds, _ = synth(H, N, C, seed=5)
    preds[3] = preds[0]                                   # duplicated models
    preds[7] = preds[0]
    preds[:, 20:40] = preds[:, 0:20]                      # duplicated items
    one = torch.zeros(C)
    one[2] = 1.0
    preds[:, 60:90] = one                                 # unanimous items
    preds = preds.cuda()
    pools = np.stack([np.random.default_rng(r).permutation(N)[:50] for r in range(4)])
    res = modelpicker_eps_search(TensorDataset(preds), epsilons=(0.5,) + SCRIPT_EPS, budget=50, seed=7,
                                 realisations=pools)
    assert res["picks"].shape == (16, 4, 50)
    assert res["pick_tie"].any() and res["best_tie"].any()
    for e in range(16):
        for r in range(4):
            assert sorted(res["picks"][e, r].tolist()) == list(range(50))     # every pool position exactly once
    _check_contract(preds, res, [(0, 0), (0, 3), (1, 1), (8, 2), (15, 0), (15, 3)])


def test_pool_is_the_whole_task_and_defaults_draw_the_script_realisations():
    from coda_b200 import TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth
    H, N, C = 9, 70, 4
    preds, _ = synth(H, N, C, seed=8)
    preds = preds.cuda()
    np.random.seed(3)
    want = np.array([np.random.permutation(N)[:N] for _ in range(3)])
    np.random.seed(3)
    torch.manual_seed(4)
    res = modelpicker_eps_search(TensorDataset(preds), epsilons=(0.4, 0.46), iterations=3, pool_size=500,
                                 budget=1000)
    assert np.array_equal(res["realisations"], want) and res["picks"].shape == (2, 3, N)
    torch.manual_seed(4)
    assert res["seed"] == int(torch.randint(0, 1 << 62, (1,)).item())
    _check_contract(preds, res, [(0, 0), (1, 2)])


def test_a_grid_larger_than_one_launch():
    from coda_b200 import TensorDataset, _native as nat
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth
    H, N, C, P, B = 6, 50, 5, 8, 8
    plan = np.zeros(5, dtype=np.int64)
    nat.check(nat.load().coda_b200_mp_runs_plan(H, 2, P, 5000, B, plan.ctypes.data))
    R = int(plan[2]) + 7
    preds, _ = synth(H, N, C, seed=9)
    preds = preds.cuda()
    np.random.seed(1)
    res = modelpicker_eps_search(TensorDataset(preds), epsilons=(0.42, 0.47), iterations=R, pool_size=P, budget=B,
                                 seed=11)
    _check_contract(preds, res, [(0, 0), (1, int(plan[2]) - 1), (0, int(plan[2])), (1, R - 1)])


def test_fp16_and_compact_slabs():
    from coda_b200 import CompactDataset, CompactSlab, TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth, synth_compact
    preds, _ = synth(24, 300, 10, seed=12)
    half = preds.half().cuda()
    np.random.seed(2)
    res = modelpicker_eps_search(TensorDataset(half), epsilons=(0.4, 0.46), iterations=3, pool_size=50, budget=30,
                                 seed=3)
    _check_contract(half, res, [(0, 0), (1, 2)])
    ids, probs, _ = synth_compact(20, 300, 40, 4, seed=13, device="cuda")
    slab = CompactSlab(ids, probs, 40)
    np.random.seed(4)
    res = modelpicker_eps_search(CompactDataset(slab), epsilons=(0.4, 0.46), iterations=3, pool_size=50, budget=30,
                                 seed=5)
    _check_contract(slab, res, [(0, 1), (1, 0)])


def test_picks_follow_modelpicker_py_while_separated():
    """A NumPy restatement of modelpicker.py's step (fp64 entropies) on the run's pool: the search's pick is the
    reference's arg-min for as long as the reference's best and runner-up entropies are apart by more than fp32 noise
    (near ties are broken by Philox here, by torch.randint there)."""
    from coda_b200 import TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth
    H, N, C = 16, 300, 8
    preds, labels = synth(H, N, C, seed=14)
    hard_all = _hard(preds)
    np.random.seed(5)
    res = modelpicker_eps_search(TensorDataset(preds.cuda()), epsilons=(0.35, 0.46, 0.49), iterations=3,
                                 pool_size=80, budget=40, seed=6, labels=labels)
    checked = 0
    for e, eps in enumerate(res["epsilons"]):
        gamma = float(np.float32((1.0 - eps) / eps))
        for r in range(3):
            pool = res["realisations"][r]
            hard, lab = hard_all[pool], labels.numpy()[pool]
            dis = (hard != hard[:, :1]).any(1)
            post = np.full(H, np.float32(1.0) / np.float32(H), dtype=np.float32)
            labeled = np.zeros(len(pool), bool)
            for s in range(40):
                cand = ~labeled & (dis if (dis & ~labeled).any() else True)
                items = np.nonzero(cand)[0]
                ent = _fp64_entropies(hard, post, C, gamma, items)
                order = np.argsort(ent, kind="stable")
                tol = _ref_tol(C, ent)
                if len(items) > 1 and ent[order[1]] - ent[order[0]] <= tol:
                    break
                pick = int(res["picks"][e, r, s])
                assert pick == int(items[order[0]]), (e, r, s)
                checked += 1
                labeled[pick] = True
                w = post * np.where(hard[pick] == lab[pick], np.float32(gamma), np.float32(1.0)).astype(np.float32)
                post = (w / np.float32(w.astype(np.float64).sum())).astype(np.float32)
    assert checked >= 20


def test_majority_labels_pool_accuracies_and_metrics_are_exact():
    from coda_b200 import TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search, search_metrics
    from coda_b200.synth import synth
    H, N, C = 40, 500, 3                                  # few classes: many equal vote counts
    preds, _ = synth(H, N, C, seed=15)
    hard = _hard(preds)
    np.random.seed(6)
    eps = (0.4, 0.45, 0.5)
    res = modelpicker_eps_search(TensorDataset(preds.cuda()), epsilons=eps, iterations=6, pool_size=100, budget=25,
                                 seed=8, threshold=0.5)
    maj = _majority(hard)
    assert np.array_equal(res["labels"], maj)
    acc = np.stack([(hard[p] == maj[p][:, None]).sum(0) for p in res["realisations"]])
    assert np.array_equal(res["pool_accuracies"], acc)
    best = res["best"]
    for e in range(len(eps)):
        success = np.array([[int(b in np.nonzero(acc[r] == acc[r].max())[0]) for b in best[e, r]] for r in range(6)])
        m = res["metrics"][float(eps[e])]
        assert m["success_mean"] == np.mean(success, axis=0).tolist()
        assert np.allclose(m["acc_mean"], np.mean([[acc[r, b] / 100 for b in best[e, r]] for r in range(6)], axis=0),
                           rtol=0, atol=1e-15)
    assert list(res["metrics"]) == [0.4, 0.45, 0.5]
    assert (res["best_avg"], res["best_fast"]) == search_metrics(best, acc, 100, eps, 0.5)[:2]


def test_refusals_before_any_launch():
    from coda_b200 import TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth
    preds, _ = synth(4, 50, 3, seed=1)
    ds = TensorDataset(preds.cuda())
    for bad in ((0.0, 0.4), (0.4, 1.0), (-0.1,), (1.5,)):
        with pytest.raises(ValueError):
            modelpicker_eps_search(ds, epsilons=bad, iterations=2, pool_size=10, budget=5)
    with pytest.raises(NotImplementedError):
        modelpicker_eps_search(TensorDataset(torch.zeros(1025, 4, 2, device="cuda")), iterations=2, pool_size=4)
    with pytest.raises(NotImplementedError):
        modelpicker_eps_search(TensorDataset(preds[:, :30].cuda(), n_offset=0, n_global=50), iterations=2,
                               pool_size=10)
    with pytest.raises(ValueError):
        modelpicker_eps_search(ds, realisations=np.array([[0, 1, 50]]))
