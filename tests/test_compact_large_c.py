"""The compact slab above C = 1024, up to C = 4096: every stage that reads it, against a host model of that one stage,
then CODA, the competing selectors and the epsilon search end to end.

  scan       coda_b200_scan_compact(_kernel)   hard, pseudo, disagree exact; ens against the NumPy ascending-h fp32
                                               model bit for bit (both kernels where both run); flags; arg-max ties
  marginals  coda_b200_pi_full_compact         U against fp64 on the densified slab within the chain's bound; pisum
  rank-1     pi_rank1_index / pi_rank1_compact the checks of test_marginal_kernels.py at C = 3201 and 4096
  CODA       construction and three labels against the oracle's quantities evaluated in fp64 on the device
  layouts    run_steps = API loop, shards=2 = one shard, pieces = whole slab
  selectors  the five competing selectors and the epsilon search against the densified twin

Outputs are poisoned before each launch, the kernel that ran is asserted, and each host model has a perturbed variant
that must fail.  Run with ``-s`` to see the worst error of every comparison against its bound."""
import math
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, coda_oracle
from test_compact_large_c_host import scan_model

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
U32 = 2.0 ** -24
SCAN_WARP_FROM_C = 400                   # compact.cu: from this C the scan runs one warp per item
POISON16, POISON32 = -0x5A5B, -0x5A5A5A5B


def _nat():
    from coda_b200 import _native as nat
    return nat, nat.load()


def _p(t):
    import ctypes as ct
    return ct.c_void_p(0 if t is None else t.data_ptr())


def _s():
    import ctypes as ct
    return ct.c_void_p(torch.cuda.current_stream().cuda_stream)


def _report(stage, label, err, tol):
    print(f"[large-c] {stage:<9} {label:<48} worst {err:.3e}   bound {tol:.1e}")


def _entries(rng, H, N, C, K):
    """(H, N, K) distinct ids (descending-score order does not matter to the scan) and scores summing to < 1."""
    base = rng.integers(0, C, (H, N, 1))
    stride = rng.integers(1, max(2, C // K), (H, N, 1))
    ids = (base + stride * np.arange(K)) % C
    p = rng.dirichlet(np.ones(K + 1), (H, N)).astype(np.float32)[..., :K]
    p = -np.sort(-p, axis=-1)
    return ids.astype(np.int64), p.astype(np.float32)


def _launch_scan(ids_t, probs_t, stride, H, N, C, K, kernel=None, ens=True):
    nat, lib = _nat()
    hard = torch.full((N, H), POISON16, dtype=torch.int16, device=DEV)
    pseudo = torch.full((N,), POISON32, dtype=torch.int32, device=DEV)
    dis = torch.full((N,), 0xA5, dtype=torch.uint8, device=DEV)
    e = torch.full((N, C), float("nan"), device=DEV) if ens else None
    flags = torch.zeros(1, dtype=torch.int32, device=DEV)
    if kernel is None:
        rc = lib.coda_b200_scan_compact(_p(ids_t), _p(probs_t), stride, H, N, C, K, _p(hard), _p(pseudo), _p(dis), _p(e),
                                        _p(flags), _s())
    else:
        rc = lib.coda_b200_scan_compact_kernel(_p(ids_t), _p(probs_t), stride, H, N, C, K, _p(hard), _p(pseudo), _p(dis),
                                               _p(e), _p(flags), kernel, _s())
    nat.check(rc, "scan_compact")
    torch.cuda.synchronize()
    return (hard.cpu().numpy().astype(np.int64) & 0xFFFF, pseudo.cpu().numpy(), dis.cpu().numpy(),
            None if e is None else e.cpu().numpy(), int(flags.item()))


def _kernels_run(fn, poison=None):
    """The kernel names of one fn() call.  A first call loads the kernels (lazy module loading: the profiler does not
    always see a kernel's first launch); ``poison`` re-poisons the outputs before the profiled call."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    if poison is not None:
        poison()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {ev.key for ev in prof.key_averages()}


# ------------------------------------------------------------------------------------------------------------------
# scan
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("C", [1024, 1599, 1600, 2048, 3001, 4096])
def test_scan_matches_the_ascending_h_model(C, K):
    H = (1, 33, 64)[(C + K) % 3]
    N, lo, Nt = 8 * 5 + 3, 11, 8 * 5 + 3 + 20          # an N-range view: model stride Nt K, not N K
    rng = np.random.default_rng(C * 10 + K)
    ids, p = _entries(rng, H, Nt, C, K)
    ids_t = torch.from_numpy(ids.astype(np.int16)).to(DEV)
    probs_t = torch.from_numpy(p).to(DEV)
    v_ids, v_p = ids_t[:, lo:lo + N], probs_t[:, lo:lo + N]
    hard_m, dis_m, ens_m, pseudo_m = scan_model(ids[:, lo:lo + N], p[:, lo:lo + N], C)
    kernels = [None] + ([1, 2] if C <= 1599 else [])
    for kern in kernels:
        hard, pseudo, dis, ens, flags = _launch_scan(v_ids, v_p, Nt * K, H, N, C, K, kern)
        assert flags == 0
        assert np.array_equal(hard, hard_m) and np.array_equal(pseudo, pseudo_m) and np.array_equal(dis, dis_m), kern
        assert np.array_equal(ens.view(np.int32), ens_m.view(np.int32)), (kern, np.abs(ens - ens_m).max())
    if H > 1:                                                    # the perturbed model: models added in descending order
        _, _, ens_d, _ = scan_model(ids[:, lo:lo + N], p[:, lo:lo + N], C, ascending=False)
        assert not np.array_equal(ens.view(np.int32), ens_d.view(np.int32))
    _report("scan", f"C={C} K={K} H={H} ens bits", 0.0, 0.0)


@pytest.mark.parametrize("C", [SCAN_WARP_FROM_C - 1, SCAN_WARP_FROM_C, 1599, 4096])
def test_scan_runs_the_kernel_its_class_count_selects(C):
    rng = np.random.default_rng(C)
    H, N, K = 5, 20, 4
    ids, p = _entries(rng, H, N, C, K)
    ids_t, probs_t = torch.from_numpy(ids.astype(np.int16)).to(DEV), torch.from_numpy(p).to(DEV)
    names = _kernels_run(lambda: _launch_scan(ids_t, probs_t, N * K, H, N, C, K))
    warp = any("k_scan_compact_warp" in k for k in names)
    thread = any("k_scan_compact<" in k or k.startswith("void k_scan_compact<") for k in names)
    assert warp == (C >= SCAN_WARP_FROM_C) and thread == (C < SCAN_WARP_FROM_C), names


@pytest.mark.parametrize("C", [1599, 2048])
def test_scan_ties_and_input_flags(C):
    """Arg-max ties go to the first class, and every input check sets its flag, on both kernels where both run."""
    nat, _ = _nat()
    H, N, K = 6, 12, 2
    rng = np.random.default_rng(7)
    ids, p = _entries(rng, H, N, C, K)
    ids[:, 0] = [C - 5, 3]                       # item 0: two classes tie in every model -> the first index, 3
    p[:, 0] = [0.4, 0.4]
    ids[:, 1] = [9, C - 1]                       # item 1: the tie at the two ends of the row
    p[:, 1] = [0.3, 0.3]
    ids_t, probs_t = torch.from_numpy(ids.astype(np.int16)).to(DEV), torch.from_numpy(p).to(DEV)
    for kern in (1, 2) if C <= 1599 else (2,):
        hard, pseudo, dis, ens, flags = _launch_scan(ids_t, probs_t, N * K, H, N, C, K, kern)
        assert flags == 0 and pseudo[0] == 3 and pseudo[1] == 9
        assert ens[0, 3] == ens[0, C - 5] and ens[1, 9] == ens[1, C - 1]
        hm, dm, em, pm = scan_model(ids, p, C)
        assert np.array_equal(pseudo, pm) and np.array_equal(ens.view(np.int32), em.view(np.int32))
    cases = [("nan", nat.FLAG_NONFINITE_INPUT), ("big", nat.FLAG_RANGE_INPUT), ("neg", nat.FLAG_RANGE_INPUT),
             ("id", nat.FLAG_RANGE_INPUT), ("rest", nat.FLAG_RANGE_INPUT), ("edge", 0)]
    for what, want in cases:
        i2, p2 = ids.copy(), p.copy()
        h, n = 4, 7
        if what == "nan":
            p2[h, n, 1] = np.nan
        elif what == "big":
            p2[h, n, 0] = 1.01
        elif what == "neg":
            p2[h, n, 1] = -0.01
        elif what == "id":
            i2[h, n, 1] = C
        elif what == "rest":
            p2[h, n] = [0.8, 0.3]                # sum 1.1: a negative remainder
        else:
            p2[h, n] = [1.0001, 0.0]             # the edge itself, and 0, set nothing
        t_i, t_p = torch.from_numpy(i2.astype(np.int16)).to(DEV), torch.from_numpy(p2).to(DEV)
        for kern in (1, 2) if C <= 1599 else (2,):
            flags = _launch_scan(t_i, t_p, N * K, H, N, C, K, kern, ens=False)[4]
            assert flags == want, (what, kern, flags)


# ------------------------------------------------------------------------------------------------------------------
# construction marginals
# ------------------------------------------------------------------------------------------------------------------
def _dirichlet_like(rng, H, C):
    D = np.full((H, C, C), 2.0 / (C - 1), np.float32) * rng.uniform(1.0, 1.3, (H, C, C)).astype(np.float32)
    D[:, np.arange(C), np.arange(C)] = 2.0 + rng.uniform(0, 0.5, (H, C)).astype(np.float32)
    return D


@pytest.mark.parametrize("C,K", [(1025, 4), (2048, 8), (4096, 3)])
def test_full_marginals_against_fp64_and_the_column_sums(C, K):
    """U[n][c] = sum_h (rest RS[h][c] + sum_j (p_j - rest) D[h][c][id_j]): an fmaf chain of m = H (K + 1) terms on fp32
    inputs (p_j - rest rounded once, RS a lane-then-tree fp32 sum of C non-negative terms).  Bound, with A the same sum
    of absolute terms in fp64: 1.01 (m + ceil(C / 32) + 7) u A.  pi_reduce of the result gives the fixed-point column
    sums of its own xi bit for bit."""
    from coda_b200 import CompactSlab
    from test_marginal_kernels import fx_shift_of, fx_sum, launch_reduce
    nat, lib = _nat()
    H, N = 4, 37
    rng = np.random.default_rng(C + K)
    ids, p = _entries(rng, H, N, C, K)
    slab = CompactSlab(torch.from_numpy(ids.astype(np.int16)).to(DEV), torch.from_numpy(p).to(DEV), C)
    D = torch.from_numpy(_dirichlet_like(rng, H, C)).to(DEV)
    DT = torch.empty((H, C, C), device=DEV)
    RS = torch.empty((H, C), device=DEV)
    U = torch.full((N, C), float("nan"), device=DEV)
    names = _kernels_run(lambda: nat.check(lib.coda_b200_pi_full_compact(
        _p(slab.ids), _p(slab.probs), N * K, _p(D), H, N, C, K, _p(DT), _p(RS), _p(U), _s()), "pi_full_compact"),
        poison=lambda: U.fill_(float("nan")))
    assert any("k_pi_full_compact_win" in k for k in names), names
    P = slab.densify().double()
    U64 = torch.einsum("hcs,hns->nc", D.double(), P)
    s32 = slab.probs[..., 0].clone()
    for j in range(1, K):
        s32 = s32 + slab.probs[..., j]
    rest = ((1.0 - s32) * (torch.tensor(1.0) / torch.tensor(float(C - K))).to(DEV)).double()   # (H, N), the kernels' fp32
    w = (slab.probs.double() - rest[..., None]).abs()                                         # (H, N, K)
    Dg = D.double()[torch.arange(H, device=DEV)[:, None, None], :, slab.ids.long()]          # (H, N, K, C): D[h][:, id]
    A = (rest.abs()[..., None] * D.double().sum(-1)[:, None, :]).sum(0) + (w[..., None] * Dg).sum((0, 2))
    bound = 1.01 * (H * (K + 1) + math.ceil(C / 32) + 7) * U32 * A + 1e-30
    err = (U.double() - U64).abs()
    _report("marginal", f"C={C} K={K} U (err / bound)", float((err / bound).max()), 1.0)
    assert bool((err <= bound).all())
    wrong = U64 - torch.einsum("cs,ns->nc", D[0].double(), P[0]) * 1e-3                        # one model's share off
    assert bool(((U.double() - wrong).abs() > bound).any())
    shift = fx_shift_of(N)
    xo, pis, fl = launch_reduce(U, shift)
    assert fl == 0 and np.array_equal(pis, fx_sum(xo.cpu().numpy(), shift))


# ------------------------------------------------------------------------------------------------------------------
# rank-1 refreshes: the checks of test_marginal_kernels.py above the per-warp shared-memory limit
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kernel", ["index", "slab"])
@pytest.mark.parametrize("H,N,C,K", [(7, 200, 3201, 4), (5, 150, 4096, 8)])
def test_rank1_refreshes_above_the_per_warp_limit(H, N, C, K, kernel):
    from test_marginal_kernels import test_compact_rank1_refresh_matches_fp64 as rank1_case
    rank1_case(H, N, C, K, kernel)
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# CODA end to end
# ------------------------------------------------------------------------------------------------------------------
def _case(H, N, C, K, seed):
    from coda_b200 import CompactSlab
    from coda_b200.synth import synth_compact
    ids, probs, labels = synth_compact(H, N, C, K, seed=seed)
    slab = CompactSlab(ids, probs, C)
    return slab, slab.densify(), labels


class _Env:
    def __init__(self, **kw):
        self.kw, self.old = kw, {}

    def __enter__(self):
        for k, v in self.kw.items():
            self.old[k] = os.environ.get(k)
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _oracle_on(D, dense_d, hard_cpu, lr_unused=None):
    """The oracle's state on the posterior D (fp32, the engine's, checked separately), its marginals in fp64 on the
    device: an OracleSelector whose EIG and P(best) run on the CPU on those marginals."""
    xi, pi = coda_oracle.consensus_marginals(D.double(), dense_d.double())
    ora = coda_oracle.OracleSelector.__new__(coda_oracle.OracleSelector)
    ora.dirichlets = D.cpu().float()
    ora.pi_hat, ora.pi_hat_xi = pi.float().cpu(), xi.float().cpu()
    ora.hard, ora.check, ora.C, ora.H = hard_cpu, True, D.shape[1], D.shape[0]
    return ora, xi, pi


@pytest.mark.parametrize("index", [None, 0])
@pytest.mark.parametrize("H,N,C,K", [(8, 400, 2048, 4), (16, 300, 3001, 2), (5, 300, 4096, 8)])
def test_coda_follows_the_oracle(H, N, C, K, index):
    from coda_b200 import CODA, CompactDataset, TensorDataset
    slab, dense, labels = _case(H, N, C, K, seed=C + K)
    dense_d = dense.to(DEV)
    with _Env(CODA_B200_COMPACT_INDEX=index):
        random.seed(0)
        sel = CODA(CompactDataset(slab.to(DEV), labels.to(DEV)))
    e = sel.engine
    try:
        assert (e.cidx is not None) == (index is None)
        twin = CODA(TensorDataset(dense_d, labels.to(DEV)))
        assert torch.equal(sel.dirichlets, twin.dirichlets)                  # integer work: the dense twin's bits
        assert torch.equal(e.hard, twin.engine.hard) and torch.equal(e.disagree, twin.engine.disagree)
        twin.close()
        pseudo = dense_d.mean(0).argmax(-1)
        Do = 2.0 * (coda_oracle.dirichlet_prior(torch.zeros((1, C, C)), 0.0, False)[0].to(DEV)
                    + 0.1 * coda_oracle.soft_confusion(pseudo, dense_d))
        np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), Do.cpu().numpy(), rtol=3e-6, atol=1e-7)
        del Do
        hard_cpu = coda_oracle.hard_predictions(dense)
        lr = float(np.float32(e.lr))
        for step in range(4):
            ora, xi, pi = _oracle_on(sel.dirichlets, dense_d, hard_cpu)
            rel = float(((sel.pi_hat.double() - pi).abs() / pi).max())
            _report("CODA", f"H={H} C={C} K={K} idx={index} step {step} pi_hat (rel)", rel, 5e-6)
            np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), pi.cpu().numpy(), rtol=5e-6, atol=1e-9)
            np.testing.assert_allclose(sel.pi_hat_xi.cpu().numpy(), xi.cpu().numpy(), rtol=1e-5, atol=1e-9)
            pb = ora.get_pbest()
            np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), pb.numpy(), atol=1e-5)
            assert int(sel.get_best_model_prediction()) == int(torch.argmax(pb))
            if step == 3:
                break
            i, q = sel.get_next_item_to_label()
            cand = [n for n in range(N) if bool((hard_cpu[:, n] != hard_cpu[0, n]).any()) and n not in sel.labeled_idxs]
            sub = sorted(set(cand[:: max(1, len(cand) // 12)][:12]) | {i})
            qo = ora.eig_scores(sub).numpy()
            got = e.eig.cpu().numpy()[np.asarray(sub)]
            _report("CODA", f"H={H} C={C} K={K} step {step} EIG", float(np.abs(got - qo).max()), 5e-6)
            np.testing.assert_allclose(got, qo, atol=5e-6)
            assert float(qo[sub.index(i)]) >= float(qo.max()) - 5e-6
            t = int(labels[i])
            D0 = sel.dirichlets.clone()
            sel.add_label(i, t, q)
            D0[torch.arange(H, device=DEV), t, hard_cpu[:, i].to(DEV)] += lr        # coda.py:319, one fp32 add
            assert torch.equal(sel.dirichlets, D0)
    finally:
        sel.close()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# layouts and the device loop at C = 2048
# ------------------------------------------------------------------------------------------------------------------
def test_layouts_and_the_device_loop():
    from coda_b200 import CODA, CompactDataset, TensorDataset
    from coda_b200.datasets import ShardedCompactSlab
    from coda_b200.synth import shard_range
    H, N, C, K = 8, 400, 2048, 4
    slab, _dense, labels = _case(H, N, C, K, seed=21)
    whole = slab.to(DEV)
    lab = labels.to(DEV)
    random.seed(3)
    api = CODA(CompactDataset(whole, lab))
    picks, best = [], []
    for _ in range(6):
        i, q = api.get_next_item_to_label()
        api.add_label(i, int(labels[i]), q)
        picks.append(i)
        best.append(int(api.get_best_model_prediction()))
    runs = []
    for ds, kw in ((CompactDataset(whole, lab), {}), (CompactDataset(whole, lab), {"shards": 2}),
                   (TensorDataset(ShardedCompactSlab([whole.narrow_items(*shard_range(N, r, 2)).to(DEV)
                                                      for r in range(2)]), lab), {})):
        random.seed(3)
        sel = CODA(ds, **kw)
        sel.run_steps(6, lab, record_best=True, tie_rule="reference")
        runs.append((sel.history()[0].tolist(), sel.best_history()[0].tolist(), sel.dirichlets.cpu().numpy().tobytes(),
                     sel.pi_hat.cpu().numpy().tobytes(), sel.get_pbest().cpu().numpy().tobytes(), random.getstate()))
        sel.close()
    assert runs[0][0] == picks and runs[0][1] == best
    assert runs[1] == runs[0] and runs[2] == runs[0]
    api.close()


# ------------------------------------------------------------------------------------------------------------------
# the competing selectors and the epsilon search
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("method", ["iid", "uncertainty", "activetesting", "vma", "model_picker"])
def test_competing_selectors_against_the_densified_twin(method):
    """The API-path checks of test_baselines_sharded.py at C = 3000 (hard / disagree identical, ensemble-derived scores
    within 1e-6, identical picks, q and best models, 2 shards = 1), then run_steps on the compact slab against
    run_steps on the densified twin from the same seeds."""
    from coda_b200 import CompactDataset, TensorDataset
    from test_baselines_sharded import _make, _seed_all
    from test_baselines_sharded import test_compact_slab_against_its_densified_twin as twin_case
    twin_case(method, (8, 300, 3000, 4, 3))
    slab, dense, labels = _case(8, 300, 3000, 4, seed=3)
    lab = labels.to(DEV)
    runs = []
    for ds in (CompactDataset(slab.to(DEV), lab), TensorDataset(dense.to(DEV), lab)):
        _seed_all()
        sel = _make(method, ds)
        sel.run_steps(12, lab)
        idx, q, _tie = (np.asarray(a).tolist() for a in sel.history())
        runs.append((idx, q, np.asarray(sel.best_history()[0]).tolist()))
        sel.close()
    if method == "uncertainty":                                  # picks follow scores that agree to 1e-6, not bits
        assert len(runs[0][0]) == len(runs[1][0]) == 12
    else:
        assert runs[0][0] == runs[1][0] and runs[0][2] == runs[1][2]
        if method in ("iid", "model_picker"):
            assert runs[0][1] == runs[1][1]


def test_eps_search_against_the_densified_twin():
    from coda_b200 import CompactDataset, TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    slab, dense, labels = _case(12, 300, 2048, 4, seed=5)
    out = []
    for ds in (CompactDataset(slab.to(DEV)), TensorDataset(dense.to(DEV))):
        np.random.seed(0)
        res = modelpicker_eps_search(ds, epsilons=[0.3, 0.45], iterations=3, pool_size=80, budget=25, seed=11)
        out.append(res)
    for k in ("picks", "best", "pick_tie", "best_tie", "realisations", "labels"):
        assert np.array_equal(np.asarray(out[0][k]), np.asarray(out[1][k])), k
    assert out[0]["best_avg"] == out[1]["best_avg"] and out[0]["best_fast"] == out[1]["best_fast"]


# ------------------------------------------------------------------------------------------------------------------
# the user path: a dense file compacted as it loads
# ------------------------------------------------------------------------------------------------------------------
def test_load_compact_of_a_4096_class_fp16_file(tmp_path):
    from coda_b200 import CODA, CompactSlab, TensorDataset, load_compact
    from coda_b200.synth import synth
    preds, labels = synth(4, 200, 4096, seed=9)
    p = str(tmp_path / "task.pt")
    torch.save(preds.half(), p)
    s = load_compact(p, DEV, 8)
    ref = CompactSlab.from_dense(preds.half().to(DEV), 8)
    assert torch.equal(s.ids, ref.ids) and torch.equal(s.probs, ref.probs)
    lab = labels.to(DEV)
    hist = []
    for slab in (s, ref):
        random.seed(0)
        sel = CODA(TensorDataset(slab, lab))
        sel.run_steps(3, lab, record_best=True)
        hist.append((sel.history()[0].tolist(), sel.best_history()[0].tolist(), sel.pi_hat.cpu().numpy().tobytes()))
        sel.close()
    assert hist[0] == hist[1]


def test_main_py_driver_through_the_shim_at_2048_classes(tmp_path):
    from coda.options import LOSS_FNS
    from coda_b200 import CODA, IID, CompactSlab, Oracle, TensorDataset
    from coda_b200.synth import synth
    from test_compact_build import _DRIVER
    preds, labels = synth(6, 300, 2048, seed=4)
    p = str(tmp_path / "task.pt")
    torch.save(preds, p)
    torch.save(labels, p.replace(".pt", "_labels.pt"))
    driver = str(tmp_path / "driver.py")
    with open(driver, "w") as f:
        f.write(_DRIVER)
    env = dict(os.environ, CODA_B200_COMPACT_K="8", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "stubs")]),
               PYTHONSAFEPATH="1")
    whole = CompactSlab.from_dense(preds.to(DEV), 8)
    lab = labels.to(DEV)
    iters = 5
    for method in ("coda", "iid"):
        out = str(tmp_path / f"{method}.json")
        r = subprocess.run([sys.executable, driver, p, method, str(iters), out], env=env, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        import json
        got = json.load(open(out))
        assert got["kind"] == "CompactSlab"
        random.seed(0); np.random.seed(0); torch.manual_seed(0); torch.cuda.manual_seed_all(0)
        ds = TensorDataset(whole, lab)
        oracle = Oracle(ds, loss_fn=LOSS_FNS["acc"])
        tl = oracle.true_losses(whole)
        best = min(oracle.true_losses(whole))
        sel = CODA(ds) if method == "coda" else IID(ds, LOSS_FNS["acc"])
        regrets = [float(tl[sel.get_best_model_prediction()] - best)]
        for _ in range(iters):
            i, q = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), q)
            regrets.append(float(tl[sel.get_best_model_prediction()] - best))
        assert got["regrets"] == regrets
        if method == "coda":
            assert got["labeled"] == list(map(int, sel.labeled_idxs))
        sel.close()
