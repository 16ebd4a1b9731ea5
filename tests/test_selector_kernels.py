"""Kernel-level tier of the competing selectors (csrc/baselines.cu, csrc/bl_ref.cu): each kernel against a host model of
tests/test_selector_kernels_host.py, evaluated on the exact inputs the kernel received (``hard``, ``ens``, the
posterior, ``labeled`` and ``disagree`` built as device tensors or read back from the scan that produced them).

  static     coda_b200_static_scores           ActiveTesting / VMA scores, bit for bit, H <= 1024, C <= 4096
  entropy    coda_b200_mp_entropy(_dev)         long double model, 1/2 fp32 ulp + fp64 bound; masked items +inf
  uncert     baselines.ensemble_entropy         fp64 on the exact ens / H, the bound of an fp32 sum over C terms
  select     weighted_total / weighted_draw / select_extreme / select_kth (one shard) with real-valued inputs
  loop       coda_b200_bl_step over thousands of steps: counts, s1 / s2, hist_loss, the posterior bits, hist_best
  tie set    coda_b200_bl_step and coda_b200_bl_best_ref on crafted LURE sums, exact ties and one-ulp neighbours

Outputs are filled with NaN or poison words before every launch, and every stage shows once that its comparison fails
against a perturbed model.  Run with ``-s`` to see the worst error of every comparison against its bound."""
import bisect
import itertools
import math
import random

import numpy as np
import pytest
import torch

from test_selector_kernels_host import (crafted_rows, entropy_ld, entropy_tol, clamped_loop_entropy, gamma_of,
                                        lure_bound, lure_exact, lure_risk, lure_sums, lure_t, normalised,
                                        boundary_distance, posterior_step, posteriors, report, static_exact, U32)
from test_baselines_loop_host import tie_pick

NAN = float("nan")
POISON = -0x5A5A5A5B
HS = (1, 2, 31, 32, 33, 255, 256, 257, 1000, 1024)
CS = (2, 3, 100, 1025, 4096)
GRID = [(H, C) for H in HS for C in CS]


def _nat():
    from coda_b200 import _native as nat
    return nat, nat.load()


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


def sweep_items():
    """Items per grid sweep of the one-warp-per-item kernels: min(ceil(N / 8), 8 · SMs) blocks of 8 warps."""
    return 8 * 8 * torch.cuda.get_device_properties(0).multi_processor_count


def craft_ens(hard, C, H, rng):
    """ens [N][C] fp32 in [0, H] with l = 0 and l = 1 on the first rows' classes."""
    N = hard.shape[0]
    ens = (rng.random((N, C)) * H).astype(np.float32)
    ens[0, hard[0, 0]] = np.float32(H)
    if N > 1:
        ens[1, hard[1, 0]] = 0.0
    return ens


# ------------------------------------------------------------------------------------------------------------------
# stage 1: static scores
# ------------------------------------------------------------------------------------------------------------------
def launch_static(hard_d, ens_d, H, N, C, want_at, want_vma):
    nat, lib = _nat()
    at = torch.full((N,), NAN, device="cuda") if want_at else None
    vma = torch.full((N,), NAN, device="cuda") if want_vma else None
    nat.check(lib.coda_b200_static_scores(_p(hard_d), _p(ens_d), H, N, C, _p(at), _p(vma), _s()), "static_scores")
    torch.cuda.synchronize()
    return (None if at is None else at.cpu().numpy()), (None if vma is None else vma.cpu().numpy())


def check_static(hard_d, ens_d, H, C, label, perturb=False):
    """Both outputs, each alone, against static_exact on ens[n, hard[n, h]] read back from the device."""
    N = hard_d.shape[0]
    hard64 = hard_d.long() & 0xFFFF
    g = torch.gather(ens_d, 1, hard64).cpu().numpy()
    at_ref, vma_ref = static_exact(g, H)
    a2, v2 = launch_static(hard_d, ens_d, H, N, C, True, True)
    a1, _ = launch_static(hard_d, ens_d, H, N, C, True, False)
    _, v1 = launch_static(hard_d, ens_d, H, N, C, False, True)
    bad = 0
    for got, ref in ((a2, at_ref), (a1, at_ref), (v2, vma_ref), (v1, vma_ref)):
        bad += int((got.view(np.uint32) != ref.view(np.uint32)).sum())
    report("static", f"{label} (items not bit-equal)", float(bad), 0)
    assert bad == 0, (label, bad)
    if perturb:                      # the model without the fp32 rounding of e / H must fail somewhere
        l64 = 1.0 - g.astype(np.float64) / H
        at_p = l64.sum(1).astype(np.float32)
        assert (at_p.view(np.uint32) != a2.view(np.uint32)).any()


@pytest.mark.gpu
@pytest.mark.parametrize("H,C", GRID)
def test_static_scores_bit_exact(H, C):
    rng = np.random.default_rng(H * 7919 + C)
    N = 160
    hard, _ = crafted_rows(H, C, N, rng)
    ens = craft_ens(hard, C, H, rng)
    hard_d = torch.from_numpy(hard.astype(np.int16)).cuda()
    check_static(hard_d, torch.from_numpy(ens).cuda(), H, C, f"H={H} C={C} N={N}", perturb=(H, C) == (257, 100))


@pytest.mark.gpu
@pytest.mark.parametrize("H,C", [(33, 100), (640, 4096), (1024, 4096)])
def test_static_scores_over_several_grid_sweeps(H, C):
    """N beyond two sweeps of the grid with a ragged tail; H = 640 and 1024 take the >48 KB shared-memory opt-in."""
    rng = np.random.default_rng(H)
    N = 2 * sweep_items() + 8 * 37 + 5
    hard = torch.from_numpy(crafted_rows(H, C, 64, rng)[0].astype(np.int16)).cuda()
    hard = torch.cat([hard, torch.randint(0, min(C, 6), (N - 64, H), dtype=torch.int16, device="cuda")])
    hard[-1] = torch.arange(H, dtype=torch.int16, device="cuda") % C          # the last item: K = min(H, C)
    ens = torch.rand((N, C), device="cuda") * H
    check_static(hard, ens, H, C, f"H={H} C={C} N={N} (sweeps)")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f32", "f16", "bf16", "compact"])
def test_static_scores_on_the_scans_ens(fmt):
    """The real scan of each slab format, then the kernel on the hard and ens it produced."""
    from coda_b200 import CompactSlab
    from coda_b200.baselines import _DeviceState
    from coda_b200.synth import synth
    H, N, C = 48, 3000, 100
    preds, _ = synth(H, N, C, 4, device="cuda")
    dt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "compact": torch.float32}[fmt]
    preds = preds.to(dt)
    if fmt == "compact":
        preds = CompactSlab.from_dense(preds, 4)
    st = _DeviceState(preds)
    hard, _dis, ens = st.scan(ens=True)
    check_static(hard, ens, H, C, f"scan {fmt} H={H} C={C}")


# ------------------------------------------------------------------------------------------------------------------
# stage 2: ModelPicker entropies
# ------------------------------------------------------------------------------------------------------------------
def launch_entropy(hard_d, post_d, H, C, gamma, labeled_d, dis_d, mask, dev_word=None):
    nat, lib = _nat()
    N = hard_d.shape[0]
    ent = torch.full((N,), NAN, device="cuda")
    if dev_word is None:
        nat.check(lib.coda_b200_mp_entropy(_p(hard_d), _p(post_d), H, N, C, gamma, _p(labeled_d), _p(dis_d), int(mask),
                                           _p(ent), _s()), "mp_entropy")
    else:
        w = torch.tensor([dev_word], dtype=torch.int64, device="cuda")
        nat.check(lib.coda_b200_mp_entropy_dev(_p(hard_d), _p(post_d), H, N, C, gamma, _p(labeled_d), _p(dis_d), _p(w),
                                               _p(ent), _s()), "mp_entropy_dev")
    torch.cuda.synchronize()
    return ent.cpu().numpy()


def check_entropy(hard, post, C, eps, ent, items, label, perturb=False):
    H = hard.shape[1]
    gm = gamma_of(eps)
    worst = worst_rel = 0.0
    for n in items:
        v, K = entropy_ld(hard[n], post, C, gm)
        tol = entropy_tol(v, post, H, K, gm)
        err = abs(float(ent[n]) - float(v))
        worst, worst_rel = max(worst, err), max(worst_rel, err / tol)
        assert err <= tol, (label, n, float(ent[n]), float(v), tol)
        if perturb:
            bad = float(v) * (1 + 4 * U32)
            assert abs(float(ent[n]) - bad) > entropy_tol(bad, post, H, K, gm) or v == 0
            perturb = False
    report("entropy", f"{label} (error / bound)", worst_rel, 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("H,C", GRID)
def test_mp_entropy_matches_long_double(H, C):
    rng = np.random.default_rng(H * 31 + C)
    i = GRID.index((H, C))
    eps = (0.35, 0.46, 0.49, 0.5)[i % 4]
    kind = ("uniform", "peaked", "subnormal")[i % 3]
    post = posteriors(H, rng)[kind]
    N = 96
    hard, _ = crafted_rows(H, C, N, rng)
    hard_d = torch.from_numpy(hard.astype(np.int16)).cuda()
    post_d = torch.from_numpy(post).cuda()
    labeled = np.zeros(N, np.uint8)
    labeled[5::7] = 1
    dis = (hard != hard[:, :1]).any(1).astype(np.uint8)
    lab_d, dis_d = torch.from_numpy(labeled).cuda(), torch.from_numpy(dis).cuda()
    for mask, word in ((0, None), (1, None), (None, 0), (None, 3)):
        m = bool(word) if word is not None else bool(mask)
        ent = launch_entropy(hard_d, post_d, H, C, gamma_of(eps), lab_d, dis_d, mask or 0, word)
        masked = (labeled == 1) | (m & (dis == 0))
        assert np.all(np.isposinf(ent[masked])) and np.all(np.isfinite(ent[~masked]))
        items = np.nonzero(~masked)[0]
        if mask == 0 and word is None:
            check_entropy(hard, post, C, eps, ent, items, f"H={H} C={C} eps={eps} {kind}", perturb=(H, C) == (33, 100))
            if H * C <= 257 * 1025:                         # the literal clamped loop on a few items
                for n in items[:2]:
                    lit = clamped_loop_entropy(hard[n], post, C, gamma_of(eps))
                    assert abs(float(ent[n]) - lit) <= H * 4e-11 + 2 * float(np.spacing(np.float32(abs(lit)) or 1e-30))
        else:
            ref = launch_entropy(hard_d, post_d, H, C, gamma_of(eps), lab_d, torch.ones_like(dis_d), 0)
            assert np.array_equal(ent[items], ref[items])       # unmasked items: the same bits as without the mask


@pytest.mark.gpu
def test_mp_entropy_over_several_grid_sweeps():
    rng = np.random.default_rng(11)
    H, C = 257, 1025
    N = 2 * sweep_items() + 8 * 11 + 3
    hard = rng.integers(0, 5, (N, H)).astype(np.int16)
    post = posteriors(H, rng)["subnormal"]
    ent = launch_entropy(torch.from_numpy(hard).cuda(), torch.from_numpy(post).cuda(), H, C, gamma_of(0.46),
                         torch.zeros(N, dtype=torch.uint8, device="cuda"), torch.ones(N, dtype=torch.uint8, device="cuda"), 0)
    sw = sweep_items()
    items = sorted(set(list(range(8)) + [sw - 1, sw, 2 * sw - 1, 2 * sw] + list(range(N - 12, N)) +
                       rng.integers(0, N, 40).tolist()))
    check_entropy(hard, post, C, 0.46, ent, items, f"H={H} C={C} N={N} (sweeps)")


# ------------------------------------------------------------------------------------------------------------------
# stage 3: Uncertainty's score
# ------------------------------------------------------------------------------------------------------------------
def check_uncertainty(ens_d, H, label, perturb=False):
    from coda_b200.baselines import ensemble_entropy
    got = ensemble_entropy(ens_d, H).cpu().numpy().astype(np.float64)
    e = ens_d.cpu().numpy().astype(np.float64)
    m = (e.astype(np.float32) / np.float32(H)).astype(np.float64)         # the exact fp32 mean torch computes first
    t = m * np.log(m + 1e-8)
    ref = -t.sum(1)
    C = e.shape[1]
    bound = (C + 4) * U32 * (np.abs(t).sum(1) + m.sum(1) + 1e-8 * C)
    err = np.abs(got - ref)
    report("uncert", f"{label} (error / bound)", float((err / bound).max()), 1.0)
    assert (err <= bound).all()
    if perturb:
        bad = -(m * np.log(m + 1e-6)).sum(1)
        assert (np.abs(got - bad) > bound).any()


@pytest.mark.gpu
@pytest.mark.parametrize("C", [2, 100, 1025, 4096])
def test_uncertainty_score_on_crafted_ens(C):
    H = 64
    ens = torch.rand((2000, C), device="cuda")
    ens = ens / ens.sum(1, keepdim=True) * H
    ens[0] = 0
    ens[0, 0] = H                                   # one certain item: entropy ~0
    ens[1] = H / C                                  # uniform: entropy log C
    check_uncertainty(ens, H, f"H={H} C={C}", perturb=C == 100)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["f16", "compact"])
def test_uncertainty_score_on_the_scans_ens(fmt):
    from coda_b200 import CompactSlab
    from coda_b200.baselines import _DeviceState
    from coda_b200.synth import synth
    H, N, C = 40, 3000, 1025
    preds, _ = synth(H, N, C, 6, device="cuda")
    preds = CompactSlab.from_dense(preds, 4) if fmt == "compact" else preds.half()
    _h, _d, ens = _DeviceState(preds).scan(ens=True)
    check_uncertainty(ens, H, f"scan {fmt} H={H} C={C}")


# ------------------------------------------------------------------------------------------------------------------
# stage 4: selection primitives
# ------------------------------------------------------------------------------------------------------------------
def sel_buffers(N):
    nat, lib = _nat()
    nb = int(lib.coda_b200_select_blocks(N))
    return dict(pf=torch.full((2 * nb,), NAN, dtype=torch.float64, device="cuda"),
                pi=torch.full((2 * nb,), POISON, dtype=torch.int64, device="cuda"),
                total=torch.full((2,), NAN, dtype=torch.float64, device="cuda"),
                out=torch.full((4,), POISON, dtype=torch.int64, device="cuda"),
                flags=torch.zeros(1, dtype=torch.int32, device="cuda"))


def draw_case(N, rng, kind):
    w = (rng.random(N) ** 3).astype(np.float32) + np.float32(1e-7)
    w[rng.random(N) < 0.1] = 0
    labeled = rng.random(N) < 0.15
    if kind == "tail_zero":
        w[-min(N - 1, 5000):] = 0                    # zero weights up to the end (several chunks)
        w[0] = max(w[0], np.float32(0.5))
    if kind == "chunks_labeled" and N > 3 * 4096:
        labeled[4096:3 * 4096] = True               # whole selection chunks labeled
    if kind == "last_only":
        labeled[:] = True
    labeled[-1] = False
    if w[~labeled].sum() == 0:
        w[-1] = 1.0
    return w, labeled


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 4095, 4096, 4097, 3 * 4096 + 1, 1_000_003])
def test_weighted_total_and_draw_with_real_weights(N):
    nat, lib = _nat()
    rng = np.random.default_rng(N)
    kinds = ["plain", "tail_zero", "chunks_labeled", "last_only"]
    draws = max(2600 // len(kinds), 1)
    excluded = checked = perturbed = 0
    for kind in kinds:
        w, labeled = draw_case(N, rng, kind)
        b = sel_buffers(N)
        w_d, lab_d = torch.from_numpy(w).cuda(), torch.from_numpy(labeled.astype(np.uint8)).cuda()
        nat.check(lib.coda_b200_weighted_total_xchg(_p(w_d), _p(lab_d), N, _p(b["pf"]), _p(b["total"]), None,
                                                    _p(b["flags"]), _s()), "weighted_total_xchg")
        total, count = b["total"].cpu().tolist()
        unl = ~labeled
        assert count == float(unl.sum())
        fs = math.fsum(float(x) for x in w[unl])
        assert abs(total - fs) <= N * 2.0 ** -53 * fs, (total, fs)
        unl_idx, wn = normalised(w, labeled, total)
        cum_unl = list(itertools.accumulate(float(x) for x in wn))
        random.seed(N + len(kind))
        for _ in range(draws):
            u = random.random()
            b["out"].fill_(POISON)
            nat.check(lib.coda_b200_weighted_draw_xchg(_p(w_d), _p(lab_d), N, _p(b["total"]), u, 0, _p(b["pf"]),
                                                       _p(b["out"]), None, _p(b["flags"]), _s()), "weighted_draw_xchg")
            pos, item, qb = b["out"][:3].tolist()
            rp = bisect.bisect(cum_unl, u * (cum_unl[-1] + 0.0), 0, len(cum_unl) - 1)       # random.choices
            if boundary_distance(cum_unl, rp, u) <= 1e-12:
                excluded += 1
                continue
            checked += 1
            assert (pos, item) == (rp, int(unl_idx[rp])), (kind, u, pos, item, rp)
            assert np.uint32(qb) == wn[rp].view(np.uint32)
            q_bad = np.float32(float(w[unl_idx[rp]]) / total)           # the normalisation in fp64, rounded once
            perturbed += int(q_bad.view(np.uint32) != wn[rp].view(np.uint32))
        assert int(b["flags"].item()) == 0
    report("select", f"N={N} draws checked / excluded near a boundary", float(excluded), checked)
    assert checked >= draws
    if N >= 4096:
        assert perturbed > 0                        # q without the fp32 total is another model


def extreme_case(N, rng, kind):
    vals = np.array([0.125, -1.5, 3.25, 7.0, np.float32(np.pi), -0.0, 0.0, np.inf], np.float32)
    v = vals[rng.integers(0, len(vals), N)]
    real = rng.random(N) < 0.3
    v[real] = rng.standard_normal(int(real.sum())).astype(np.float32)
    labeled = rng.random(N) < 0.2
    if kind == "all_labeled":
        labeled[:] = True
    if kind == "all_inf":
        v[~labeled] = np.inf
    if kind == "zeros":
        v[:] = np.where(rng.random(N) < 0.5, np.float32(-0.0), np.float32(0.0))
    return v.astype(np.float32), labeled


@pytest.mark.gpu
@pytest.mark.parametrize("N", [1, 4095, 4097, 3 * 4096 + 1, 1_000_003])
def test_select_extreme_and_kth_with_real_scores(N):
    nat, lib = _nat()
    rng = np.random.default_rng(N + 1)
    for kind in ("mixed", "all_labeled", "all_inf", "zeros"):
        v, labeled = extreme_case(N, rng, kind)
        for want_max in (0, 1):
            b = sel_buffers(N)
            v_d, lab_d = torch.from_numpy(v).cuda(), torch.from_numpy(labeled.astype(np.uint8)).cuda()
            best = torch.full((4,), POISON, dtype=torch.int64, device="cuda")
            nat.check(lib.coda_b200_select_extreme_xchg(_p(v_d), _p(lab_d), N, want_max, _p(b["pi"]), _p(best), None,
                                                        _p(b["flags"]), _s()), "select_extreme_xchg")
            bits, cnt, lower, mine = best.tolist()
            unl = ~labeled
            if not unl.any():
                assert cnt == 0 and mine == 0
                ref_ties = np.zeros(0, np.int64)
            else:
                ext = v[unl].max() if want_max else v[unl].min()
                ref_ties = np.nonzero(unl & (v == ext))[0]
                got = np.uint32(bits & 0xFFFFFFFF).view(np.float32)
                assert got == ext and (ext != 0 or got == 0), (kind, got, ext)
                assert (cnt, lower, mine) == (len(ref_ties), 0, len(ref_ties))
            ks = sorted(set([0, 1, len(ref_ties) // 2, len(ref_ties) - 1, len(ref_ties)]))
            for k in ks:
                if k < 0:
                    continue
                out = torch.full((1,), POISON, dtype=torch.int64, device="cuda")
                nat.check(lib.coda_b200_select_kth_xchg(_p(v_d), _p(lab_d), N, _p(b["pi"]), _p(best), k, 0, _p(out),
                                                        None, _p(b["flags"]), _s()), "select_kth_xchg")
                want = int(ref_ties[k]) if k < len(ref_ties) else -1
                assert int(out.item()) == want, (kind, want_max, k)
    report("select", f"N={N} extreme / kth (mismatches)", 0.0, 0)


# ------------------------------------------------------------------------------------------------------------------
# stage 5: the host-free loop's state over long runs
# ------------------------------------------------------------------------------------------------------------------
SEED = 987654321


def loop_run(cls, H, N, C, steps, data_seed, **kw):
    from coda.options import accuracy_loss
    from coda_b200 import TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, data_seed, device="cuda")
    ds = TensorDataset(preds, labels)
    sel = cls(ds, **kw) if cls.__name__ == "ModelPicker" else cls(ds, accuracy_loss)
    random.seed(0)
    sel.run_steps(steps, labels, seed=SEED)
    st = sel.state
    assert int(st.ls[1].item()) == steps, "the device loop stopped early"
    hard = (st.hard.long() & 0xFFFF).cpu().numpy()
    lab = labels.cpu().numpy()
    idx = st.h_idx[:steps].cpu().numpy()
    return sel, st, hard, lab, idx


def expected_best(rv, M, purpose=1):
    """hist_best of a step: the Philox pick (purpose 1, counter M) among the exact minima of rv."""
    ties = np.nonzero(rv == rv.min())[0]
    j = tie_pick(SEED, M, purpose, len(ties)) if len(ties) > 1 else 0
    return int(ties[j]), int(len(ties) > 1)


@pytest.mark.gpu
@pytest.mark.parametrize("method", ["IID", "Uncertainty"])
def test_loop_counts_and_best_model(method):
    import coda_b200.baselines as bl
    steps = 3000
    sel, st, hard, lab, idx = loop_run(getattr(bl, method), 64, 5000, 10, steps, 21)
    L = (hard[idx] != lab[idx][:, None]).astype(np.int64)
    cum = np.cumsum(L, 0)
    assert np.array_equal(st.counts.cpu().numpy(), cum[-1])
    hb, ht = st.h_best[:steps].cpu().numpy(), st.h_btie[:steps].cpu().numpy()
    ties = 0
    for s in range(steps):
        b, t = expected_best(cum[s], s + 1)
        assert (hb[s], ht[s]) == (b, t), (method, s)
        ties += t
    report("loop", f"{method} {steps} steps: hist_best exact (tie steps)", float(ties), steps)
    wrong = sum(expected_best(cum[s], s + 1, purpose=0)[0] != hb[s] for s in range(steps))
    assert wrong > 0                                          # the item draws' Philox stream picks other ties


@pytest.mark.gpu
@pytest.mark.parametrize("method,H,N,steps", [("ActiveTesting", 32, 3000, 2500), ("VMA", 32, 3000, 2000),
                                              ("ActiveTesting", 16, 600, 600)])
def test_loop_lure_sums_and_best_model(method, H, N, steps):
    import coda_b200.baselines as bl
    sel, st, hard, lab, idx = loop_run(getattr(bl, method), H, N, 10, steps, 22)
    L = hard[idx] != lab[idx][:, None]
    assert np.array_equal(st.h_loss[:steps].cpu().numpy().astype(bool), L)
    q = st.h_q[:steps].cpu().numpy()
    assert np.array_equal(q, q.astype(np.float32).astype(np.float64))          # recorded fp32 q, widened
    s1, s2 = st.s1.cpu().numpy(), st.s2.cpu().numpy()
    assert np.array_equal(s1, L.sum(0).astype(np.float64))
    r1, r2 = lure_sums(N, q, L)
    assert np.array_equal(s2.view(np.int64), r2.view(np.int64))               # the running sum, bit for bit
    hb = st.h_best[:steps].cpu().numpy()
    a1, a2 = np.zeros(H), np.zeros(H)
    wrong_plain = 0
    for s in range(steps):
        t = lure_t(float(N), float(s + 1), float(q[s]))
        a1 = a1 + np.where(L[s], 1.0, 0.0)
        a2 = a2 + np.where(L[s], t, 0.0)
        rv = np.array([lure_risk(x, y, float(N), float(s + 1)) for x, y in zip(a1, a2)])
        b, _ = expected_best(rv, s + 1)
        assert hb[s] == b, (method, s)
        plain = (a1 + (N - s - 1) * a2) / (s + 1)
        wrong_plain += expected_best(plain, s + 1)[0] != b
    ex = lure_exact(N, list(q), L)
    exf = np.array([float(v) for v in ex])
    bound = lure_bound(N, list(q), s1, s2)
    err = np.abs(rv - exf)
    report("loop", f"{method} H={H} N={N} m={steps}: risk vs rational LURE", float(err.max()), float(bound.max()))
    assert (err <= bound).all()
    order = np.argsort(exf)
    if H > 1 and exf[order[1]] - exf[order[0]] > 2 * bound.max():
        assert hb[-1] == order[0]
    if steps == N:                                                         # m = N: the plain mean
        assert np.array_equal(rv, s1 / N) and all(v == sum(L[:, h]) / N for h, v in enumerate(exf))
    report("loop", f"{method} H={H}: best models a non-fma model would get wrong", float(wrong_plain), steps)


@pytest.mark.gpu
def test_loop_modelpicker_posterior_bits_and_entropy():
    import coda_b200.baselines as bl
    # gamma = 3: with gamma < 2 the normalising sum stays below 2 and the smallest subnormal 2^-149 divided by it rounds
    # back to 2^-149, so no posterior ever reaches 0; here the weak models underflow to subnormals and then to 0
    H, N, C, steps, eps = 1024, 4000, 10, 3000, 0.25
    sel, st, hard, lab, idx = loop_run(bl.ModelPicker, H, N, C, steps, 23, epsilon=eps)
    g32 = np.float32(sel.gamma)
    post = np.full(H, np.float32(1.0) / np.float32(H), np.float32)
    torch_post = post.copy()
    counts = np.zeros(H, np.int64)
    for s in range(steps):
        agree = hard[idx[s]] == lab[idx[s]]
        post = posterior_step(post, agree, g32)
        nxt = torch.from_numpy(torch_post) * (float(g32) ** torch.from_numpy(agree).float())
        torch_post = (nxt / nxt.sum()).numpy()
        counts += agree
        b, _ = expected_best(-counts, s + 1)
        assert st.h_best[s].item() == b, s
    got = st.lpost.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), post.view(np.uint32))
    assert not np.array_equal(torch_post.view(np.uint32), got.view(np.uint32))    # torch's fp32 sum is another model
    assert np.array_equal(st.counts.cpu().numpy(), counts)
    dis = st.disagree.cpu().numpy()
    assert int(st.ls[7].item()) == int(dis.sum()) - int(dis[idx].sum())
    sub = int(((got > 0) & (got < np.finfo(np.float32).tiny)).sum())
    zero = int((got == 0).sum())
    report("loop", f"ModelPicker H={H} {steps} steps: subnormal / zero posteriors", float(sub), zero)
    assert sub >= 2 and zero >= 1
    # stage 2 on this posterior: the kernel's entropies of the unlabeled items against long double
    labeled = st.labeled
    ent = launch_entropy(st.hard, st.lpost, H, C, float(g32), labeled, st.disagree, 1)
    unl = np.nonzero(labeled.cpu().numpy() == 0)[0]
    rng = np.random.default_rng(0)
    items = [n for n in rng.choice(unl, 60, replace=False) if dis[n]]
    check_entropy(hard, got, C, eps, ent, items, f"long-run posterior H={H}")


# ------------------------------------------------------------------------------------------------------------------
# the best model's tie set: bl_step and bl_best_ref on crafted LURE sums
# ------------------------------------------------------------------------------------------------------------------
def crafted_lure(H, Ng, m, rng):
    """s1, s2 [H] whose risks fl(fma(Ng - m, s2, s1) / m) hold exact ties between different (s1, s2), neighbours one ulp
    above the minimum, and at least one model on which a multiply-then-add would decide the tie differently."""
    base = lure_risk(3.0, 0.0123, Ng, m)
    up = math.nextafter(base, math.inf)
    cand = {}                                             # (fma risk, multiply-then-add risk) -> sums
    for a in map(float, range(12)):
        c = 0.0123 + (3.0 - a) / (Ng - m)
        for k in range(-300, 301):
            y = c + k * np.spacing(c)
            r, plain = lure_risk(a, y, Ng, m), (a + (Ng - m) * y) / m
            if r in (base, up) and plain in (base, up):
                cand.setdefault((r, plain), []).append((a, y))
    pick = cand.get((base, base), [])[:6] + cand.get((base, up), [])[:2] + cand.get((up, up), [])[:6] + \
        cand.get((up, base), [])[:2]
    assert cand.get((base, up)) or cand.get((up, base)), "no sums on which the contraction decides a tie"
    x1 = [a for a, _ in pick]
    x2 = [y for _, y in pick]
    while len(x1) < H:                                    # the rest well above
        x1.append(float(rng.integers(6, 20))); x2.append(float(rng.uniform(0.02, 0.05)))
    p = rng.permutation(H)
    return np.array(x1)[p], np.array(x2)[p]


@pytest.mark.gpu
def test_best_model_tie_set_of_bl_step_and_bl_best_ref():
    nat, lib = _nat()
    import ctypes
    from coda_b200.baselines import torch_rng_words
    H, Nloc, Ng, m = 40, 4, 1000, 10
    rng = np.random.default_rng(12)
    s1, s2 = crafted_lure(H, float(Ng), float(m), rng)
    rv = np.array([lure_risk(a, b, float(Ng), float(m)) for a, b in zip(s1, s2)])
    ties = np.nonzero(rv == rv.min())[0]
    plain = (s1 + (Ng - m) * s2) / m
    assert len(ties) > 2 and not np.array_equal(np.nonzero(plain == plain.min())[0], ties)
    dev = "cuda"
    z = lambda n, dt: torch.zeros(n, dtype=dt, device=dev)
    hard = z((Nloc, H), torch.int16)
    labels = z(Ng, torch.int64)                          # every model right on the item: the sums do not move
    T = dict(labeled=z(Nloc, torch.uint8), dis=z(Nloc, torch.uint8), ls=z(16, torch.int64),
             best=z(4, torch.int64), pick=z(3, torch.int64), total=z(2, torch.float64), counts=z(H, torch.int32),
             s1=torch.from_numpy(s1).to(dev), s2=torch.from_numpy(s2).to(dev), hidx=z(1, torch.int64),
             hq=z(1, torch.float64), htie=z(1, torch.int32), hbest=z(1, torch.int32), hbt=z(1, torch.int32),
             hloss=z((1, H), torch.uint8), flags=z(1, torch.int32), trng=z(625, torch.int32), grng=z(2, torch.int64))
    a = nat.BlLoopStruct()
    a.method, a.H, a.N, a.n_offset, a.n_global = nat.BL_ACTIVETESTING, H, Nloc, 0, Ng
    a.hard, a.disagree, a.labeled, a.labels = _p(hard), _p(T["dis"]), _p(T["labeled"]), _p(labels)
    a.pre, a.ls, a.best, a.pick, a.total = None, _p(T["ls"]), _p(T["best"]), _p(T["pick"]), _p(T["total"])
    a.counts, a.s1, a.s2, a.post, a.gamma, a.hist_cap = _p(T["counts"]), _p(T["s1"]), _p(T["s2"]), None, 1.0, 1
    a.hist_idx, a.hist_q, a.hist_tie = _p(T["hidx"]), _p(T["hq"]), _p(T["htie"])
    a.hist_best, a.hist_best_tie, a.hist_loss, a.flags = _p(T["hbest"]), _p(T["hbt"]), _p(T["hloss"]), _p(T["flags"])
    q_bits = int(np.float32(0.001).view(np.uint32))
    step_seen, ref_seen = set(), set()
    for trial in range(24):
        seed = 1000 + trial
        T["ls"].zero_()
        T["ls"][0] = m - 1
        T["ls"][6] = seed
        T["pick"].copy_(torch.tensor([0, 0, q_bits]))
        T["hbest"].fill_(POISON)
        nat.check(lib.coda_b200_bl_step(ctypes.byref(a), None, _s()), "bl_step")
        torch.cuda.synchronize()
        assert np.array_equal(T["s1"].cpu().numpy(), s1) and np.array_equal(T["s2"].cpu().numpy(), s2)
        j = tie_pick(seed, m, 1, len(ties))
        assert int(T["hbest"].item()) == int(ties[j]) and int(T["hbt"].item()) == 1
        step_seen.add(int(T["hbest"].item()))
        # bl_best_ref after that step: torch.randperm(cnt)[0] on the CPU generator, from the replica of its state
        torch.manual_seed(trial)
        T["trng"].copy_(torch_rng_words(torch.get_rng_state()))
        T["hbest"].fill_(POISON)
        nat.check(lib.coda_b200_bl_best_ref(ctypes.byref(a), _p(T["trng"]), _p(T["grng"]), _s()), "bl_best_ref")
        torch.cuda.synchronize()
        torch.manual_seed(trial)
        want = int(ties[int(torch.randperm(len(ties))[0])])
        assert int(T["hbest"].item()) == want, trial
        ref_seen.add(want)
    pties = np.nonzero(plain == plain.min())[0]
    wrong = sum(int(pties[tie_pick(1000 + t, m, 1, len(pties))]) != int(ties[tie_pick(1000 + t, m, 1, len(ties))])
                if len(pties) > 1 else 1 for t in range(24))
    report("tie set", f"{len(ties)} ties of {H}; picks seen bl_step / bl_best_ref", float(len(step_seen)), len(ref_seen))
    assert wrong > 0 and step_seen <= set(ties.tolist()) and ref_seen <= set(ties.tolist())
