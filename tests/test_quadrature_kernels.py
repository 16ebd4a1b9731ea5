"""Kernel-level tier of the EIG quadrature: every stage of the per-step EIG chain against an fp64 NumPy model of the
same stage, evaluated on the exact inputs the stage received (the engine's own D, grid, tables, masks, m0, pi_hat, U,
entry lists and gains).  Each comparison therefore measures one kernel's error, not what earlier stages pass on.

  stage 1  coda_b200_beta_tables            dL, G0T, G1T, PB and the bf16 limb tables dLb / Gb   (tables.cu)
  stage 2  k_pair_rows_tc / k_pair_rows     P(best | hypothetical) rows and their gains          (pairs_tc.cu, pairs.cu)
  stage 3  k_row_gains<NQ> / k_row_gains_any  gains from the cached rows                          (gain.cu)
  stage 4  k_eig_assemble_g8 / k_gain_eig   eig and the block arg-max records                     (gain.cu)
  stage 5  k_step_mixture                   m0, H_before, best model                              (step.cu)
  stage 6  incremental state                the class-t refresh leaves what a full rebuild writes, bit for bit

Every output under test is filled with NaN before its launch (only the entries the kernel is documented to write), every
test asserts the kernel path it ran, and every stage shows once that its comparison fails on a perturbed model.  The
fp64 model is anchored to the reference by the CPU tests at the top (its quadrature known answers and the goldens'
initial P(best)).  Run with ``-s`` to see the worst error of every comparison."""
import contextlib
import os

import numpy as np
import pytest
import torch
from scipy.special import gammaln

from helpers import GOLDEN, golden_names, load_golden

P = 256                                  # quadrature nodes
U32 = 2.0 ** -24                         # fp32 unit roundoff
CDF_FLOOR = float(np.float32(1e-30))     # the reference's cdf / normaliser floor, an fp32 constant
NAN = float("nan")
POISON = 0x7FC00000                      # int64 words of the records: NaN bits, a huge index, a huge count

# budgets of the bf16-limb tensor-core rows and the fp32 SIMT rows (tests/test_limb_precision_model.py)
TC_ROW_ATOL, TC_GAIN_ATOL, F32_GAIN_ATOL = 6e-6, 1e-7, 5e-8
EIG_ATOL = 5e-6                          # EIG parity tolerance against the reference (tests/test_gpu_parity.py)
# tables are built in fp64 and rounded to fp32 once: 4 ulps relative, above a floor that covers the fp64 noise of
# dL = L_hit - L_miss near x = 1 (both logs ~0) and fp32 denormals of G / PB
TAB_RTOL, DL_FLOOR, G_FLOOR = 4 * U32, 1e-9, 1e-40


def _report(stage, label, err, tol):
    print(f"[quadrature] {stage:<9} {label:<34} worst {err:.3e}   tolerance {tol:.1e}")


# ------------------------------------------------------------------------------------------------------------------
# fp64 model
# ------------------------------------------------------------------------------------------------------------------
def quad_grid():
    """coda.py:86: the fp32 torch.linspace grid (its bits are not those of np.linspace rounded to fp32)."""
    return torch.linspace(1e-6, 1 - 1e-6, P).numpy()


def trap_weights(x32):
    """Trapezoid weight of every node from the fp32 grid differences, as tables.cu forms them."""
    d = (x32[1:] - x32[:-1]).astype(np.float64)                       # fp32 differences
    return 0.5 * (np.concatenate([[0.0], d]) + np.concatenate([d, [0.0]]))


def beta_params(D, classes):
    """(alpha, beta), each (len(classes), H) fp32, of the class Betas of an (H, C, C) fp32 posterior: the row sum
    accumulated exactly and rounded once to fp32, beta = rowsum - alpha in fp32 (coda.py:24, tables.cu)."""
    cls = np.asarray(classes)
    rs = D[:, cls, :].astype(np.float64).sum(-1).astype(np.float32)  # (H, R); exact before the rounding
    alpha = D[:, cls, cls]
    return alpha.T.copy(), (rs - alpha).astype(np.float32).T.copy()


def tables64(alpha, beta, w=1.0, wq=None):
    """fp64 model of coda_b200_beta_tables for R classes.  alpha, beta: (R, H) fp32.  Returns dL (R, H, P),
    G0 / G1 (R, H, P) and PB (R, H).  The fp32 roundings the kernels share with the reference are mirrored (grid,
    grid differences, 1 - x, a - 1, a + b, a + w, b + w, the 1e-30f floors); everything else is fp64."""
    x32 = quad_grid()
    d = (x32[1:] - x32[:-1]).astype(np.float64)
    wq = trap_weights(x32) if wq is None else wq
    lx, l1x = np.log(x32.astype(np.float64)), np.log((np.float32(1) - x32).astype(np.float64))
    a, b, w = np.asarray(alpha, np.float32), np.asarray(beta, np.float32), np.float32(w)
    pdf, L = [], []
    for va, vb in ((a, b), (a, b + w), (a + w, b)):                  # before, miss (coda.py:166), hit (coda.py:165)
        am1, bm1 = (va - np.float32(1)).astype(np.float64), (vb - np.float32(1)).astype(np.float64)
        lgn = gammaln((va + vb).astype(np.float64)) - (gammaln(va.astype(np.float64)) + gammaln(vb.astype(np.float64)))
        p = np.exp(am1[..., None] * lx + bm1[..., None] * l1x + lgn[..., None])
        cdf = np.zeros_like(p)
        np.cumsum(0.5 * (p[..., 1:] + p[..., :-1]) * d, axis=-1, out=cdf[..., 1:])
        pdf.append(p)
        L.append(np.log(np.maximum(cdf, CDF_FLOOR)))
    (pb, pm, ph), (Lb, Lm, Lh) = pdf, L
    S0, SB = Lm.sum(-2, keepdims=True), Lb.sum(-2, keepdims=True)
    loo = lambda v: np.exp(np.clip(v, -80.0, 80.0))                   # coda.py:107
    raw = (wq * pb * loo(SB - Lb)).sum(-1)
    return dict(dL=Lh - Lm, G0=wq * pm * loo(S0 - Lm), G1=wq * ph * loo(S0 - Lh),
                PB=raw / np.maximum(raw.sum(-1, keepdims=True), CDF_FLOOR))


def tables_of(D, classes, w=1.0, wq=None):
    """tables64 of the given classes of an (H, C, C) posterior, in chunks of classes (bounded memory)."""
    H = D.shape[0]
    step = max(1, 4096 // H)
    parts = [tables64(*beta_params(D, classes[i:i + step]), w=w, wq=wq) for i in range(0, len(classes), step)]
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def ent64(m):
    q = np.maximum(m, 1e-12)                                          # coda.py:254
    return -q * np.log2(q)


def gain64(PH, PB, m0, pic):
    """Information gain of rows PH (M, H) of classes with 'before' rows PB (M, H), weights pic (M,) (coda.py:274-276)."""
    return (ent64(m0)[None] - ent64(m0[None] + pic[:, None] * (PH - PB))).sum(1)


def gain_arith_bound(PH, PB, m0, pic):
    """Bound of the fp32 evaluation of gain64 as the kernels do it (ent_term, common.cuh): per model the two entropy
    terms (ent_bound), the rounding of m0 + pic (ph - PB) times |f'|, the rounded difference f(m0) - f(mix), and a
    chain of at most H / 32 + 8 additions of those differences.
    __log2f's 2^-22 absolute error near m = 1 makes this ~3e-7 whenever one model holds most of P(best): far above
    the fp64-gain budget of the rows, far below the 5e-6 EIG tolerance."""
    mix = m0[None] + pic[:, None] * (PH - PB)
    q = np.maximum(np.abs(mix), 1e-12)
    per = ent_bound(m0)[None] + ent_bound(mix) + np.abs(np.log2(q) + 1 / np.log(2)) * U32 * (q + pic[:, None] * np.abs(PH - PB))
    diff = np.abs(ent64(m0)[None] - ent64(mix))
    return per.sum(1) + (PH.shape[1] / 32 + 9) * U32 * diff.sum(1)


def ent_bound(m):
    """fp32 f(m) = -max(m, 1e-12) log2(max(m, 1e-12)) with __log2f (abs error <= 2^-22 on [0.5, 2], 2 ulp elsewhere)
    and one rounded product."""
    q = np.maximum(m, 1e-12)
    return q * (2.0 ** -22 + 2 * U32 * np.abs(np.log2(q))) + U32 * np.abs(ent64(m))


def rows64(Z, dL, G0, G1):
    """Normalised P(best | hypothetical) rows of one class: Z (M, H) {0, 1}, dL (H, P), G0 / G1 (P, H).
    Returns (rows, logD, D, a0, a1)."""
    logD = Z @ dL
    Dv = np.exp(logD)
    a0, a1 = Dv @ G0, Dv @ G1
    prob = np.where(Z > 0, a1, a0)
    return prob / np.maximum(prob.sum(1, keepdims=True), CDF_FLOOR), logD, Dv, a0, a1


def simt_row_bound(Z, PH, logD, Dv, a0, a1, G0, G1):
    """First-order bound of |k_pair_rows - rows64| for every entry, from the fp32 arithmetic of pairs.cu:
      phase A  logD(x) = FMA chain over the n_z models of Z; dL <= 0 (a hit Beta is stochastically larger than the
               miss Beta, so its cdf is smaller), the partial sums are monotone and the chain errs by <= n_z u |logD|;
               expf adds 2 ulp, so D(x) carries a relative error <= n_z u |logD(x)| + 2u;
      phase B  a_k[h] = sum_x G_k[x, h] D(x), a 256-term FMA chain of non-negative terms: <= 256 u relative, plus the
               D errors weighted by G_k D: n_z u <|logD|>_h, the G_k D-weighted mean over the nodes; D values below
               the fp32 normal range add <= 2^-126 sum_x G_k[x, h] absolute;
      normalise  the row sum (H / 32 terms per lane, a 5-level tree) adds (H / 32 + 5) u + max_h rel(a), the division u.
    The sum of the three relative terms, doubled for the second-order terms, is the bound."""
    H = Z.shape[1]
    nz = Z.sum(1, keepdims=True)
    wl = Dv * np.abs(logD)
    with np.errstate(divide="ignore", invalid="ignore"):
        m0 = np.where(a0 > 0, (wl @ G0) / a0, 0.0)
        m1 = np.where(a1 > 0, (wl @ G1) / a1, 0.0)
    rel_a = 258 * U32 + nz * U32 * np.where(Z > 0, m1, m0)
    s = np.where(Z > 0, a1, a0).sum(1, keepdims=True)
    under = np.where(Z > 0, G1.sum(0)[None], G0.sum(0)[None]) * 2.0 ** -126 / np.maximum(s, 1e-300)
    rel_s = (H / 32 + 5) * U32 + rel_a.max(1, keepdims=True)
    return 2 * (PH * (rel_a + rel_s + U32) + under)


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the model against the reference's own numbers
# ------------------------------------------------------------------------------------------------------------------
KAT_RTOL = 4e-6


def test_fp64_model_reproduces_the_quadrature_known_answers():
    """compute_pbest_beta_batched of the reference on extreme Betas (alpha, beta from 0.02 to 200).  The oracle test
    holds the fp32 oracle to rtol 2e-6; this fp64 model needs 4e-6 on row 0 (alpha = 200, beta = 40, the sharpest
    Beta), where the reference's own fp32 cumulative trapezoid is 3.3e-6 off the fp64 value.  The reference's
    algorithm evaluated in fp64 (the oracle on double tensors) agrees with the model to 5e-7 on every row: what is
    left is a + b, which the model rounds to fp32 as the reference and tables.cu do."""
    from helpers import coda_oracle
    z = np.load(f"{GOLDEN}/quadrature_kat.npz")
    assert np.array_equal(quad_grid(), z["grid"])
    got = tables64(z["alpha"], z["beta"])["PB"]
    o64 = coda_oracle.pbest_rows(torch.from_numpy(z["alpha"]).double(), torch.from_numpy(z["beta"]).double()).numpy()
    np.testing.assert_allclose(got, o64, rtol=5e-7, atol=0)
    _report("model", "quadrature_kat PB (rel)", float((np.abs(got - z["pbest"]) / z["pbest"]).max()), KAT_RTOL)
    np.testing.assert_allclose(got[1:], z["pbest"][1:], rtol=2e-6, atol=1e-9)
    np.testing.assert_allclose(got, z["pbest"], rtol=KAT_RTOL, atol=1e-9)


@pytest.mark.parametrize("name", [n for n in golden_names() if "h256" not in n])
def test_fp64_model_reproduces_the_goldens_initial_pbest(name):
    """P(best) = sum_c pi_hat[c] PB[c] from the goldens' initial posterior and pi_hat, at the oracle test's tolerance
    for the reference's get_pbest.  (The H = 256 golden stores no initial posterior.)"""
    g = load_golden(name)
    D = g["init_dirichlets"]
    PB = tables_of(D, np.arange(D.shape[1]))["PB"]
    m0 = g["init_pi_hat"].reshape(-1).astype(np.float64) @ PB
    ref = g["init_pbest"].reshape(-1)
    _report("model", f"{name} init_pbest", float(np.abs(m0 - ref).max()), 1e-5)
    np.testing.assert_allclose(m0, ref, rtol=1e-5, atol=1e-8)


def test_fp64_model_mirrors_the_fp32_complement_of_the_grid():
    """1 - x is formed in fp32 (as the reference and tables.cu form it): with beta in the thousands, log(1 - x) taken
    in fp64 instead moves log pdf by up to (beta - 1) * 3e-8 -- far more than the 4-ulp table tolerance."""
    x32 = quad_grid()
    exact = np.log1p(-x32.astype(np.float64))
    fp32 = np.log((np.float32(1) - x32).astype(np.float64))
    shift = 4000 * np.abs(exact - fp32).max()
    assert shift > 1e-5, shift


# ------------------------------------------------------------------------------------------------------------------
# GPU plumbing
# ------------------------------------------------------------------------------------------------------------------
def _nat():
    from coda_b200 import _native as nat
    return nat, nat.load()


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


@contextlib.contextmanager
def _env(name, value):
    old = os.environ.get(name)
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = value
    try:
        yield
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


def _selector(preds, tc=True, mode="incremental"):
    from coda_b200 import CODA, TensorDataset
    with _env("CODA_B200_TC", None if tc else "0"):
        sel = CODA(TensorDataset(preds.to("cuda:0"), None), mode=mode)
    torch.cuda.synchronize()
    return sel


def _flags_clear(e):
    torch.cuda.synchronize()
    assert int(e.flags.item()) == 0, hex(int(e.flags.item()))


def design_hard(H, C, n_base, seed, *, pool=None, straddle=True, unanimous=3, many=(), heavy=None, acc=0.7, twice=False):
    """(N, H) hard predictions built so that masks, entry counts and work-list lengths are known:
      base items      true class y from ``pool``, every model right with probability ``acc``, else one of the next
                      three classes of the pool;
      straddle items  models b - 1 and b predict one class, every other model another, for every mask-word boundary
                      b = 32 k < H (heavy rows whose mask straddles two words, and the phase-B pass boundary);
      many items      one item per k in ``many`` with exactly k distinct predicted classes;
      unanimous       items on which every model agrees (disagree = 0);
      heavy           {class: heavy rows}: unanimous items of the class are added until it has exactly that many;
      twice           every item is followed by an identical copy (exact EIG ties)."""
    rng = np.random.default_rng(seed)
    pool = np.arange(C) if pool is None else np.asarray(pool)
    y = pool[rng.integers(0, len(pool), n_base)]
    k = rng.integers(1, min(3, len(pool) - 1) + 1, (n_base, H)) if len(pool) > 1 else np.zeros((n_base, H), int)
    pos = np.searchsorted(pool, y)[:, None]
    wrong = pool[(pos + k) % len(pool)]
    rows = [np.where(rng.random((n_base, H)) < acc, y[:, None], wrong)]
    if straddle:
        for j, b in enumerate(range(32, H, 32)):
            r = np.full(H, pool[j % len(pool)])
            r[b - 1:b + 1] = pool[(j + 1) % len(pool)]
            rows.append(r[None])
    for kk in many:
        rows.append((np.arange(H) % kk)[None])
    for j in range(unanimous):
        rows.append(np.full((1, H), pool[j % len(pool)]))
    hard = np.concatenate(rows).astype(np.int64)
    if heavy:
        cnt = heavy_counts(hard, C)
        fill = []
        for c, want in heavy.items():
            assert cnt[c] <= want, (c, cnt[c], want)
            fill += [np.full((1, H), c)] * int(want - cnt[c])
        hard = np.concatenate([hard] + fill)
    if twice:
        hard = np.repeat(hard, 2, axis=0)
    return hard


def heavy_counts(hard, C):
    N = hard.shape[0]
    per = np.zeros((N, C), np.int64)
    np.add.at(per, (np.repeat(np.arange(N), hard.shape[1]), hard.ravel()), 1)
    return (per >= 2).sum(0)


def slab_from_hard(hard, C, seed=0, twice=False):
    """Post-softmax (H, N, C) fp32 slab whose arg-max is ``hard``: 0.6 on the chosen class, the other 0.4 spread
    unevenly.  ``twice``: item 2 i + 1 carries the same bytes as item 2 i."""
    N, H = hard.shape
    rng = np.random.default_rng(seed)
    p = rng.uniform(0.5, 1.5, (H, N, C)).astype(np.float32)
    hi, ni = np.arange(H)[:, None], np.arange(N)[None, :]
    p[hi, ni, hard.T] = 0
    p *= np.float32(0.4) / p.sum(-1, keepdims=True)
    p[hi, ni, hard.T] = np.float32(0.6)
    if twice:
        p[:, 1::2] = p[:, 0::2]
    return torch.from_numpy(p)


def tiles_of(e, width):
    """(class, first position, count, 0) tiles of ``width`` same-class work-list positions and the first tile of
    every class: the engine's tiling for the other row kernel."""
    base = e.cls_base_host
    per = np.diff(base)
    nt = (per + width - 1) // width
    toff = np.concatenate([[0], np.cumsum(nt)])
    cls = np.repeat(np.arange(e.C), nt)
    k = np.arange(int(toff[-1])) - toff[cls]
    start = base[cls] + width * k
    cnt = np.minimum(width, per[cls] - width * k)
    tiles = np.stack([cls, start, cnt, np.zeros_like(cnt)], 1).astype(np.int32)
    return torch.from_numpy(tiles).cuda(), torch.from_numpy(toff.astype(np.int64)).cuda()


# ---- stage launches into fresh, poisoned buffers -----------------------------------------------------------------
def limb_model_index(C, Hp):
    """Model index h of every element of dLb [C][Hp/32][3][256 x 32] and Gb [C][16][4][Hp x 16], both in the
    documented wgmma no-swizzle K-major core-matrix order [k_core][r_core][8 rows][8 elements]:
      dLb tile: rows = nodes, K = 32 models -> h = 32 kb + 8 k_core + element, x = 8 r_core + row;
      Gb tile:  rows = models, K = 16 nodes -> h = 8 r_core + row, x = 16 chunk + 8 k_core + element."""
    hd = (32 * np.arange(Hp // 32)[None, :, None, None, None, None, None]
          + 8 * np.arange(4)[None, None, None, :, None, None, None] + np.arange(8)[None, None, None, None, None, None, :])
    hd = np.broadcast_to(hd, (C, Hp // 32, 3, 4, 32, 8, 8))
    hg = 8 * np.arange(Hp // 8)[None, None, None, None, :, None, None] + np.arange(8)[None, None, None, None, None, :, None]
    hg = np.broadcast_to(hg, (C, 16, 4, 2, Hp // 8, 8, 8))
    return hd, hg


def decode_limbs(dLb, Gb, C, Hp):
    """-> d (3, C, Hp, P) limbs of dL, g (4, C, Hp, P) limbs {G0 hi, G0 lo, G1 hi, G1 lo}, as fp64."""
    a = dLb.float().cpu().numpy().reshape(C, Hp // 32, 3, 4, 32, 8, 8)       # c, kb, limb, k_core, r_core, row, el
    d = a.transpose(2, 0, 1, 3, 6, 4, 5).reshape(3, C, Hp, P)
    b = Gb.float().cpu().numpy().reshape(C, 16, 4, 2, Hp // 8, 8, 8)         # c, chunk, table, k_core, r_core, row, el
    g = b.transpose(2, 0, 4, 5, 1, 3, 6).reshape(4, C, Hp, P)
    return d.astype(np.float64), g.astype(np.float64)


def fresh_tables(H, C, limbs):
    """Output buffers of coda_b200_beta_tables, NaN wherever the kernel writes and zero in the caller's padding
    (G0T / G1T / limb columns h >= H); PB is NaN in full (k_pb_normalize writes its padding itself)."""
    Hp = (H + 31) // 32 * 32
    dev = torch.device("cuda:0")
    t = dict(dL=torch.full((C, H, P), NAN, device=dev), G0T=torch.zeros((C, P, Hp), device=dev),
             G1T=torch.zeros((C, P, Hp), device=dev), PB=torch.full((C, Hp), NAN, device=dev))
    t["G0T"][:, :, :H] = NAN
    t["G1T"][:, :, :H] = NAN
    t["dLb"] = t["Gb"] = None
    if limbs:
        hd, hg = limb_model_index(C, Hp)
        t["dLb"] = torch.from_numpy(np.where(hd < H, np.float32(NAN), np.float32(0)).reshape(C, Hp // 32, 3, 256 * 32)).to(dev, torch.bfloat16)
        t["Gb"] = torch.from_numpy(np.where(hg < H, np.float32(NAN), np.float32(0)).reshape(C, 16, 4, Hp * 16)).to(dev, torch.bfloat16)
    return t


def launch_tables(D, H, C, lo, hi, t, sel=None, w=1.0):
    nat, lib = _nat()
    grid = torch.linspace(1e-6, 1 - 1e-6, P).cuda()
    n = 1 if sel is not None else hi - lo
    scratch = torch.empty(int(lib.coda_b200_tables_scratch_bytes(H, n)), dtype=torch.uint8, device="cuda:0")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    nat.check(lib.coda_b200_beta_tables(_p(D), _p(grid), H, C, P, w, lo, hi, _p(sel), _p(scratch), _p(t["dL"]),
                                        _p(t["G0T"]), _p(t["G1T"]), _p(t["PB"]), _p(t["dLb"]), _p(t["Gb"]),
                                        _p(flags), _s()), "beta_tables")
    torch.cuda.synchronize()
    assert int(flags.item()) == 0


def tables_np(t):
    return {k: (None if v is None else v.float().cpu().numpy()) for k, v in t.items()}


def check_tables(D, classes, got, H, label, w=1.0):
    """Kernel tables (numpy, all classes) against tables64 on the kernel's own D, for ``classes``."""
    m = tables_of(D, classes, w=w)
    Hp = got["PB"].shape[1]
    ker = dict(dL=got["dL"][classes], G0=got["G0T"][classes][:, :, :H].transpose(0, 2, 1),
               G1=got["G1T"][classes][:, :, :H].transpose(0, 2, 1), PB=got["PB"][classes][:, :H])
    for k, floor in (("dL", DL_FLOOR), ("G0", G_FLOOR), ("G1", G_FLOOR), ("PB", G_FLOOR)):
        assert np.isfinite(ker[k]).all(), (label, k)
        r = (np.abs(ker[k] - m[k]) / (TAB_RTOL * np.abs(m[k]) + floor)).max()
        rel = (np.abs(ker[k] - m[k]) / np.maximum(np.abs(m[k]), floor / TAB_RTOL)).max()
        _report("tables", f"{label} {k} (rel, ulp)", float(rel), TAB_RTOL)
        assert r <= 1, (label, k, r)
    assert (got["PB"][:, H:] == 0).all() and got["PB"].shape == (D.shape[1], Hp)
    return m


def launch_rows(e, tc, gains=True, tiles=None, tile_off=None, sel=None, ph=True):
    """Row kernel over all tiles (or the ``sel`` class) into fresh NaN buffers -> (ph_cache, gain)."""
    nat, lib = _nat()
    out_ph = torch.full((e.npairs, e.Hp), NAN, device=e.dev) if ph else None
    out_g = torch.full((e.npairs,), NAN, device=e.dev) if gains else None
    if tiles is None:
        tiles, tile_off = (e.tiles, e.tile_off) if tc == e.use_tc else tiles_of(e, 128 if tc else 32)
    nt = int(tiles.shape[0]) if sel is None else int(e.max_cls_tiles if tc == e.use_tc else
                                                      torch.diff(tile_off).max().item())
    tail = (_p(e.PB), _p(e.m0) if gains else None, _p(e.pi_hat) if gains else None, e.H, _p(out_ph), _p(out_g),
            _p(sel), _p(tile_off) if sel is not None else None, _p(e.flags), _s())
    if tc:
        nat.check(lib.coda_b200_pair_rows_tc(_p(tiles), 0, nt, _p(e.zmask), _p(e.row_of), _p(e.dLb), _p(e.Gb), *tail), "rows_tc")
    else:
        nat.check(lib.coda_b200_pair_rows(_p(tiles), 0, nt, _p(e.zmask), _p(e.row_of), _p(e.dL), _p(e.G0T), _p(e.G1T),
                                          *tail), "rows")
    _flags_clear(e)
    return out_ph, out_g


def engine_np(e):
    """Host copies of what the row / gain stages read."""
    return dict(dL=e.dL.cpu().numpy().astype(np.float64), G0T=e.G0T.cpu().numpy().astype(np.float64),
                G1T=e.G1T.cpu().numpy().astype(np.float64), PB=e.PB.cpu().numpy().astype(np.float64),
                m0=e.m0.cpu().numpy().astype(np.float64), pi_hat=e.pi_hat.cpu().numpy().astype(np.float64),
                zmask=e.zmask.cpu().numpy().view(np.uint32), row_of=e.row_of.cpu().numpy().astype(np.int64))


def mask_bits(zm, H):
    b = (zm[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1
    return b.reshape(len(zm), -1)[:, :H].astype(np.float64)


def positions_to_check(e, tiles_np, seed=0):
    """Every work-list position up to H = 256; above, every heavy row, every row of one whole class, the first and
    last row of every tile and a fixed-seed sample of the rest."""
    if e.H <= 256:
        return np.arange(e.npairs)
    row_of = e.row_of.cpu().numpy()
    base = e.cls_base_host
    c = e.C // 2
    pos = [np.flatnonzero(row_of >= e.T), np.arange(base[c], base[c + 1]), tiles_np[:, 1],
           tiles_np[:, 1] + tiles_np[:, 2] - 1, np.random.default_rng(seed).choice(e.npairs, 512, replace=False)]
    return np.unique(np.concatenate(pos))


def row_models(e, E, pos, flip=None):
    """rows64 of the work-list positions ``pos`` on the engine's own tables -> per position (row id, class, model
    row, SIMT bound).  ``flip``: (position, model) whose mask bit the model flips (negative control)."""
    H = e.H
    cls = np.searchsorted(e.cls_base_host, pos, side="right") - 1
    out = []
    for c in np.unique(cls):
        q = pos[cls == c]
        Z = mask_bits(E["zmask"][q], H)
        if flip is not None and flip[0] in q:
            i = int(np.flatnonzero(q == flip[0])[0])
            Z[i, flip[1]] = 1 - Z[i, flip[1]]
        G0, G1 = E["G0T"][c][:, :H], E["G1T"][c][:, :H]
        PH, logD, Dv, a0, a1 = rows64(Z, E["dL"][c], G0, G1)
        out.append((E["row_of"][q], np.full(len(q), c), PH, simt_row_bound(Z, PH, logD, Dv, a0, a1, G0, G1)))
    rows, cl, PH, bnd = (np.concatenate(v) for v in zip(*out))
    return rows, cl, PH, bnd


def row_error(ph, rows, PH, bound=None):
    """worst |kernel - model| (or its ratio to the per-entry bound) over the rows."""
    d = np.abs(ph[rows, :PH.shape[1]].astype(np.float64) - PH)
    return float(d.max()) if bound is None else float((d / bound).max())


# ------------------------------------------------------------------------------------------------------------------
# shared engines (built once per module; the tests that label items build their own)
# ------------------------------------------------------------------------------------------------------------------
# (H, C, base items, design options): every Hp from 32 to 1024 that routes differently
ROW_CASES = {
    29: (6, 40, dict(pool=(3, 4, 5), heavy={0: 1, 1: 2, 2: 3})),     # Hp 32: class work lists of 31, 32, 33 positions
    64: (5, 30, {}),
    96: (4, 12, dict(heavy={0: 30, 1: 31, 2: 32})),                 # Hp 96, three blocks in one pass: 127, 128, 129
    128: (4, 30, {}),
    150: (4, 24, {}),                                               # Hp 160: phase B in 3 + 2 blocks
    192: (4, 24, {}),                                               # 3 + 3
    200: (4, 24, {}),                                               # Hp 224: 4 + 3
    256: (4, 24, {}),                                               # 4 + 4
    270: (4, 16, {}),                                               # SIMT from here on: Hp 288
    300: (4, 16, {}),                                               # Hp 320 (k_row_gains_any)
    384: (4, 12, {}),
    500: (4, 12, {}),                                               # Hp 512
}
_ENGINES = {}


def _case(H):
    if H not in _ENGINES:
        if H == 1024:        # configs[4]'s width: C = 100, items with 33 and 70 distinct classes, 3 table batches
            hard = design_hard(1024, 100, 24, seed=11, many=(33, 70), twice=True)
            _ENGINES[H] = _selector(slab_from_hard(hard, 100, seed=11, twice=True))
        else:
            C, nb, kw = ROW_CASES[H]
            hard = design_hard(H, C, nb, seed=H, **kw)
            _ENGINES[H] = _selector(slab_from_hard(hard, C, seed=H))
    return _ENGINES[H].engine


@pytest.fixture(scope="module", autouse=True)
def _release_engines():
    yield
    for s in _ENGINES.values():
        s.close() if hasattr(s, "close") else None
    _ENGINES.clear()
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# stage 1: tables
# ------------------------------------------------------------------------------------------------------------------
def random_posterior(H, C, seed):
    """(H, C, C) fp32 posterior whose class Betas fall in three regimes by (model, class): broad (alpha, beta in
    0.3..3), moderate (5..50) and sharp (alpha 2000..5000, beta 600..1500: the benchmark's posterior)."""
    rng = np.random.default_rng(seed)
    reg = (np.arange(H)[:, None] + 3 * np.arange(C)[None]) % 3
    lo, hi = np.array([0.3, 5.0, 2000.0])[reg], np.array([3.0, 50.0, 5000.0])[reg]
    alpha, beta = rng.uniform(lo, hi), rng.uniform(lo, hi) * np.array([1.0, 1.0, 0.3])[reg]
    D = rng.uniform(0.01, 1.0, (H, C, C))
    i = np.arange(C)
    D[:, i, i] = 0
    D *= (beta / D.sum(-1))[..., None]
    D[:, i, i] = alpha
    return D.astype(np.float32)


def bf16(v):
    return torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(torch.bfloat16).float().numpy()


def check_limbs(t, H, C):
    """The bf16 limb tables, decoded from their documented layout: dL = d0 + d1 + d2 exactly, G = hi + lo within
    2^-16, every limb the round-to-nearest bf16 of its residual, zero in the padded models."""
    Hp = (H + 31) // 32 * 32
    d, g = decode_limbs(t["dLb"], t["Gb"], C, Hp)
    assert (d[:, :, H:] == 0).all() and (g[:, :, H:] == 0).all()
    d, g = d[:, :, :H].astype(np.float32), g[:, :, :H].astype(np.float32)
    dL = t["dL"].cpu().numpy()
    assert np.array_equal(d[0].astype(np.float64) + d[1] + d[2], dL.astype(np.float64))
    assert np.array_equal(d[0], bf16(dL))
    r1 = dL - d[0]
    assert np.array_equal(d[1], bf16(r1)) and np.array_equal(d[2], bf16(r1 - d[1]))
    for hi, lo, G in ((g[0], g[1], t["G0T"]), (g[2], g[3], t["G1T"])):
        Gf = G.cpu().numpy().transpose(0, 2, 1)[:, :H]
        assert np.array_equal(hi, bf16(Gf)) and np.array_equal(lo, bf16(Gf - hi))
        # 2^-16 relative above the bf16 denormals (spacing 2^-133), where the low limb cannot carry the residual
        assert (np.abs(hi.astype(np.float64) + lo - Gf) <= 2.0 ** -16 * np.abs(Gf) + 2.0 ** -133).all()


def same_bits(a, b):
    if a is None or b is None:
        return a is None and b is None
    it = torch.int16 if a.element_size() == 2 else torch.int32
    return torch.equal(a.contiguous().view(it), b.contiguous().view(it))


TABLE_SHAPES = [(1, 3), (2, 20), (5, 7), (31, 16), (33, 5), (97, 18), (129, 4), (200, 17), (256, 12), (300, 16),
                (1024, 6)]


@pytest.mark.gpu
@pytest.mark.parametrize("H,C", TABLE_SHAPES)
def test_tables_match_the_fp64_model_and_carry_the_same_bits_in_every_launch_shape(H, C):
    """dL, G0T, G1T, PB (and the limbs wherever the tensor-core rows read them) against tables64 on the same D; the
    same bits from one launch over [0, C) (k_beta_combine split over models for C >= 16, over more CTAs below), one
    launch per class, and the device-``sel`` single-class launch of the per-step refresh."""
    Hp = (H + 31) // 32 * 32
    limbs = Hp <= 256
    Dn = random_posterior(H, C, seed=7 * H + C)
    D = torch.from_numpy(Dn).cuda()
    t = fresh_tables(H, C, limbs)
    launch_tables(D, H, C, 0, C, t)
    got = tables_np(t)
    check_tables(Dn, np.arange(C), got, H, f"H={H} C={C}")
    if limbs:
        check_limbs(t, H, C)
    per, dev = fresh_tables(H, C, limbs), fresh_tables(H, C, limbs)
    sel = torch.zeros(2, dtype=torch.int64, device="cuda:0")
    for c in range(C):
        launch_tables(D, H, C, c, c + 1, per)
        sel[1] = c
        launch_tables(D, H, C, 0, 1, dev, sel=sel)
    for k in t:
        assert same_bits(t[k], per[k]) and same_bits(t[k], dev[k]), k
    if (H, C) == (33, 5):
        # negative control: the model without the trapezoid weight of one end node
        x32 = quad_grid()
        m = tables_of(Dn, np.arange(C))
        end = -1 if max(m["G0"][..., -1].max(), m["G1"][..., -1].max()) > max(m["G0"][..., 0].max(), m["G1"][..., 0].max()) else 0
        wq = trap_weights(x32)
        wq[end] = 0.0
        bad = tables_of(Dn, np.arange(C), wq=wq)
        worst = max((np.abs(got[k + "T"].transpose(0, 2, 1)[:, :H] - bad[k]) / (TAB_RTOL * np.abs(bad[k]) + G_FLOOR)).max()
                    for k in ("G0", "G1"))
        assert worst > 1, worst


@pytest.mark.gpu
def test_tables_kernel_reproduces_the_quadrature_known_answers():
    """The reference's known answers through the kernel: H = 5 models, C = 7 classes, class c's Betas the row c of
    quadrature_kat.npz (alpha on the diagonal of D, beta in one other entry).  The kernel forms beta as
    fp32(alpha + beta) - alpha, as coda.py:24 does; the fp64 model on those inputs and the reference's P(best) must
    both hold."""
    z = np.load(f"{GOLDEN}/quadrature_kat.npz")
    H, C = 5, 7
    Dn = np.zeros((H, C, C), np.float32)
    for c in range(C):
        Dn[:, c, c] = z["alpha"][c]
        Dn[:, c, (c + 1) % C] = z["beta"][c]
    t = fresh_tables(H, C, True)
    launch_tables(torch.from_numpy(Dn).cuda(), H, C, 0, C, t)
    got = tables_np(t)
    check_tables(Dn, np.arange(C), got, H, "quadrature_kat")
    pb = got["PB"][:, :H]
    _report("tables", "quadrature_kat PB vs reference (rel)", float((np.abs(pb - z["pbest"]) / z["pbest"]).max()), KAT_RTOL)
    np.testing.assert_allclose(pb, z["pbest"], rtol=KAT_RTOL, atol=1e-9)


@pytest.mark.gpu
def test_tables_built_in_batches_carry_the_bits_of_one_launch():
    """At H = 1024 the engine builds the C = 100 class tables in batches (TABLE_BATCH_BYTES of scratch each): the
    same bits as one launch over all classes; three classes (first, first of the second batch, last) against the model."""
    e = _case(1024)
    assert e.C == 100 and e.table_batch < e.C // 2
    t = fresh_tables(e.H, e.C, False)
    launch_tables(e.D, e.H, e.C, 0, e.C, t)
    for k in ("dL", "G0T", "G1T", "PB"):
        assert same_bits(t[k], getattr(e, k)), k
    check_tables(e.D.cpu().numpy(), np.array([0, e.table_batch, e.C - 1]), tables_np(t), e.H, "H=1024 C=100 batched")


def check_padding(e):
    H = e.H
    assert (e.G0T[:, :, H:] == 0).all() and (e.G1T[:, :, H:] == 0).all() and (e.PB[:, H:] == 0).all()
    if e.use_tc:
        hd, hg = limb_model_index(e.C, e.Hp)
        assert (e.dLb.float().cpu().numpy().reshape(hd.shape)[hd >= H] == 0).all()
        assert (e.Gb.float().cpu().numpy().reshape(hg.shape)[hg >= H] == 0).all()


# ------------------------------------------------------------------------------------------------------------------
# stage 2: rows
# ------------------------------------------------------------------------------------------------------------------
def straddling_heavy_positions(e, E):
    """Work-list positions of heavy rows whose mask has bits in two different 32-model words."""
    heavy = np.flatnonzero(E["row_of"] >= e.T)
    words = (E["zmask"][heavy] != 0).sum(1)
    return heavy[words >= 2]


ROW_HS = list(ROW_CASES) + [1024]


@pytest.mark.gpu
@pytest.mark.parametrize("H", ROW_HS)
def test_rows_match_the_fp64_model_at_every_width(H):
    """Every cached row and gain of both row kernels (SIMT only above Hp = 256) against rows64 / gain64 on the engine's
    own tables, m0, pi_hat and masks: the tensor-core rows within their limb budget, the SIMT rows within the bound
    derived from their fp32 arithmetic (simt_row_bound)."""
    e = _case(H)
    Hp = (H + 31) // 32 * 32
    assert e.Hp == Hp and e.use_tc == (Hp <= 256)
    E = engine_np(e)
    per = np.diff(e.cls_base_host)
    if H == 29:
        assert per[:3].tolist() == [31, 32, 33]
    if H == 96:
        assert per[:3].tolist() == [127, 128, 129]
    if H > 32:
        assert len(straddling_heavy_positions(e, E)) >= Hp // 32 - 1
    for tc in ([True, False] if e.use_tc else [False]):
        nblk = Hp // 32
        npass = 2 if nblk > 4 else 1
        path = f"tc {(nblk + npass - 1) // npass}+{nblk - (nblk + npass - 1) // npass}" if tc else "simt"
        ph, g = launch_rows(e, tc)
        ph, g = ph.cpu().numpy(), g.cpu().numpy()
        assert np.isfinite(ph).all() and np.isfinite(g).all() and (ph[:, H:] == 0).all()
        tiles = (e.tiles if tc == e.use_tc else tiles_of(e, 128 if tc else 32)[0]).cpu().numpy()
        pos = positions_to_check(e, tiles)
        rows, cl, PH, bnd = row_models(e, E, pos)
        err = row_error(ph, rows, PH)
        if tc:
            _report("rows", f"H={H} Hp={Hp} {path}", err, TC_ROW_ATOL)
            assert err < TC_ROW_ATOL
        else:
            ratio = row_error(ph, rows, PH, bnd)
            _report("rows", f"H={H} Hp={Hp} simt (bound ratio {ratio:.2f})", err, float(bnd.max()))
            assert ratio <= 1
        gm = gain64(PH, E["PB"][cl, :H], E["m0"][:H], E["pi_hat"][cl])
        gtol = (TC_GAIN_ATOL if tc else F32_GAIN_ATOL) + gain_arith_bound(PH, E["PB"][cl, :H], E["m0"][:H], E["pi_hat"][cl])
        gerr = np.abs(g[rows] - gm)
        _report("gains", f"H={H} Hp={Hp} {path}", float(gerr.max()), float(gtol.max()))
        assert (gerr <= gtol).all()
        if H == 150:
            # negative control: one mask bit of one straddling heavy row flipped in the model
            q = int(straddling_heavy_positions(e, E)[0])
            h = int(np.flatnonzero(mask_bits(E["zmask"][[q]], H)[0])[0])
            rows2, _, PH2, bnd2 = row_models(e, E, np.array([q]), flip=(q, h))
            assert row_error(ph, rows2, PH2) > (TC_ROW_ATOL if tc else 0) and \
                (tc or row_error(ph, rows2, PH2, bnd2) > 1)


def sharp_posterior(H, C, seed):
    """cfg3-like concentrations (N = 5e5 items, 5 000 per class) with synth's confusion structure: model h is right
    with probability a_h, else one of the next three classes with 0.9 (1 - a_h), else any other class."""
    from coda_b200.synth import model_accuracies
    acc = model_accuracies(H, seed).numpy().astype(np.float64)[:, None]
    n = 5e5 / C
    i = np.arange(C)
    D = np.empty((H, C, C))
    D[:] = (1.0 / (C - 1) + n * (1 - acc) * 0.1 / (C - 4))[:, :, None]
    for k in (1, 2, 3):
        D[:, i, (i + k) % C] = 1.0 / (C - 1) + n * (1 - acc) * 0.9 / 3
    D[:, i, i] = 1.0 + n * acc
    return D.astype(np.float32)


@pytest.mark.gpu
def test_sharp_posterior_at_full_tensor_core_width():
    """The benchmark's posterior regime at H = 256, C = 100 (diagonals 2 750-4 600): tables, every row of both row
    kernels, the gains and the EIG against the fp64 model."""
    from coda_b200.synth import synth
    H, C = 256, 100
    preds, _ = synth(H, 600, C, seed=3)
    sel = _selector(preds)
    e = sel.engine
    assert e.use_tc and e.Hp == 256
    Dn = sharp_posterior(H, C, 3)
    assert 2000 < Dn[:, np.arange(C), np.arange(C)].min() and Dn[:, np.arange(C), np.arange(C)].max() < 5000
    with e._on():
        e.D.copy_(torch.from_numpy(Dn))
        e._tables(0, C)
        e._mixture()
    _flags_clear(e)
    check_tables(Dn, np.arange(C), tables_np({k: getattr(e, k) for k in ("dL", "G0T", "G1T", "PB")}), H, "sharp H=256 C=100")
    E = engine_np(e)
    rows, cl, PH, bnd = row_models(e, E, np.arange(e.npairs))
    gm = gain64(PH, E["PB"][cl, :H], E["m0"][:H], E["pi_hat"][cl])
    arith = gain_arith_bound(PH, E["PB"][cl, :H], E["m0"][:H], E["pi_hat"][cl])
    gmodel = np.empty(e.npairs)
    gmodel[rows] = gm
    eig_m = eig64(e, gmodel)[0]
    for tc in (True, False):
        ph, g = launch_rows(e, tc)
        ph, g = ph.cpu().numpy(), g.cpu().numpy()
        err, gerr = row_error(ph, rows, PH), np.abs(g[rows] - gm)
        path = "tc 4+4" if tc else "simt"
        gtol = (TC_GAIN_ATOL if tc else F32_GAIN_ATOL) + arith
        _report("rows", f"sharp H=256 {path}", err, TC_ROW_ATOL if tc else float(bnd.max()))
        _report("gains", f"sharp H=256 {path}", float(gerr.max()), float(gtol.max()))
        assert (gerr <= gtol).all()
        e.gain.copy_(torch.from_numpy(g))
        eig, _rec = launch_eig(e, e.max_entries, e.ell_row, e.ell_cls, e.ell_k)
        eerr = float(np.abs(eig.astype(np.float64) - eig_m).max())
        _report("eig", f"sharp H=256 {path} vs fp64 chain", eerr, EIG_ATOL)
        assert eerr < EIG_ATOL
        assert err < TC_ROW_ATOL if tc else row_error(ph, rows, PH, bnd) <= 1
    sel.close()


# ------------------------------------------------------------------------------------------------------------------
# stage 3: row_gains
# ------------------------------------------------------------------------------------------------------------------
def row_classes(e):
    H, T = e.H, e.T
    rc = e.row_cls.cpu().numpy().astype(np.int64) & 0xFFFF
    return np.concatenate([np.arange(T) // (1 + H), rc[: e.n_heavy]])


@pytest.mark.gpu
@pytest.mark.parametrize("H", [29, 64, 96, 128, 150, 256, 300, 384, 500, 1024])
def test_row_gains_from_the_cached_rows_match_the_fp64_model(H):
    """k_row_gains<NQ> (Hp = 128 NQ, NQ = 1..4) and k_row_gains_any (every other Hp) on the kernel's own row cache:
    the gain of every row against gain64, within the bound of its fp32 arithmetic (gain_arith_bound).  Padded models contribute nothing: the cached rows, PB and m0 are zero
    there (the kernel reads all Hp columns)."""
    e = _case(H)
    nat, lib = _nat()
    Hp = e.Hp
    nq = Hp // 128 if Hp % 128 == 0 and Hp <= 512 else 0
    variant = f"k_row_gains<{nq}>" if nq else "k_row_gains_any"
    assert variant == {128: "k_row_gains<1>", 256: "k_row_gains<2>", 384: "k_row_gains<3>",
                       512: "k_row_gains<4>"}.get(Hp, "k_row_gains_any")
    with e._on():
        e._pair_rows(0, e.ntiles, gains=False)
        e.gain.fill_(NAN)
        nat.check(lib.coda_b200_row_gains(_p(e.ph_cache), _p(e.row_cls), e.n_heavy, H, e.C, _p(e.PB), _p(e.m0),
                                          _p(e.pi_hat), _p(e.gain), _s()), "row_gains")
    _flags_clear(e)
    E = engine_np(e)
    assert (E["PB"][:, H:] == 0).all() and (E["m0"][H:] == 0).all()
    cls = row_classes(e)
    g = e.gain.cpu().numpy()
    assert len(g) == len(cls) == e.npairs and np.isfinite(g).all()
    err, tol, bad = 0.0, 0.0, 0.0
    for r0 in range(0, e.npairs, 8192):
        ph = e.ph_cache[r0:r0 + 8192].cpu().numpy().astype(np.float64)
        assert (ph[:, H:] == 0).all()
        c = cls[r0:r0 + 8192]
        bnd = gain_arith_bound(ph[:, :H], E["PB"][c, :H], E["m0"][:H], E["pi_hat"][c])
        d = np.abs(g[r0:r0 + 8192] - gain64(ph[:, :H], E["PB"][c, :H], E["m0"][:H], E["pi_hat"][c]))
        assert (d <= bnd).all()
        err, tol = max(err, float(d.max())), max(tol, float(bnd.max()))
        if r0 == 0:
            # negative control: the model with the class weight pi_hat of the next class
            cn = (c + 1) % e.C
            bad = float((np.abs(g[r0:r0 + 8192] - gain64(ph[:, :H], E["PB"][c, :H], E["m0"][:H], E["pi_hat"][cn])) / bnd).max())
    _report("rowgains", f"H={H} Hp={Hp} {variant}", err, tol)
    assert bad > 1, bad


# ------------------------------------------------------------------------------------------------------------------
# stage 4: EIG assembly and records
# ------------------------------------------------------------------------------------------------------------------
IDX_NONE = 2 ** 63 - 1


def eig64(e, gain, swap=None):
    """fp64 (sum_c U g0 + sum_e U (gain_e - g0)) / max(sum_c U, 1e-12) from the kernel's gains and U, and the bound of
    its fp32 evaluation: every kernel sums at most C + entries + 8 terms in one chain, so the error is <= (C + n_e
    + 16) u times the sum of the terms' magnitudes, over the denominator, plus the division.  ``swap``: two classes
    whose g0 the model exchanges (negative control)."""
    N, C, H = e.N, e.C, e.H
    U = e.U.cpu().numpy().astype(np.float64)
    off = e.ent_off.cpu().numpy().astype(np.int64)
    er = e.ent_row.cpu().numpy()[: off[-1]].astype(np.int64)
    ec = e.ent_cls.cpu().numpy()[: off[-1]].astype(np.int64) & 0xFFFF
    g = gain.astype(np.float64)
    g0 = g[np.arange(C) * (1 + H)]
    if swap is not None:
        g0[list(swap)] = g0[list(swap[::-1])]
    item = np.repeat(np.arange(N), np.diff(off))
    corr = U[item, ec] * (g[er] - g0[ec])
    num = U @ g0 + np.bincount(item, corr, minlength=N)
    mag = np.abs(U) @ np.abs(g0) + np.bincount(item, np.abs(corr), minlength=N)
    den = np.maximum(U.sum(1), 1e-12)
    eig = num / den
    return eig, (C + np.diff(off) + 16) * U32 * mag / den + 2 * U32 * np.abs(eig)


def host_record(eig, labeled, disagree, last=False):
    """The merged record {bits(vA), iA, |A|, bits(vB), iB, bits(v2A), bits(v2B), 0} over A = unlabeled & disagree and
    B = unlabeled: first index of the maximum, and the best value among the set's other items.  ``last``: the last
    index of the maximum instead (negative control)."""
    def best(mask):
        idx = np.flatnonzero(mask)
        if not len(idx):
            return -np.inf, IDX_NONE, -np.inf
        v = eig[idx]
        k = int(np.flatnonzero(v == v.max())[-1 if last else 0])
        rest = np.delete(v, k)
        return v[k], int(idx[k]), (rest.max() if len(rest) else -np.inf)
    bits = lambda v: int(np.float32(v).view(np.int32))
    A, B = (~labeled) & disagree, ~labeled
    vA, iA, v2A = best(A)
    vB, iB, v2B = best(B)
    return [bits(vA), iA, int(A.sum()), bits(vB), iB, bits(v2A), bits(v2B), 0]


def launch_eig(e, max_entries, ell_row, ell_cls, ell_k):
    """coda_b200_gain_eig into a NaN eig and poisoned block records, then step_merge -> (eig, merged record)."""
    nat, lib = _nat()
    with e._on():
        e.eig.fill_(NAN)
        e.partials.fill_(POISON)
        e.bestrec.fill_(POISON)
        nat.check(lib.coda_b200_gain_eig(_p(e.U), e.N, e.C, e.H, _p(e.ent_off), _p(e.ent_row), _p(e.ent_cls), _p(e.gain),
                                         _p(e.labeled), _p(e.disagree), e.n_offset, max_entries, _p(ell_row),
                                         _p(ell_cls), ell_k, _p(e.eig), _p(e.partials), _p(e.flags), _s()), "gain_eig")
        e._call("coda_b200_step_merge", e.st, None, e._s())
    _flags_clear(e)
    return e.eig.cpu().numpy(), e.bestrec.cpu().numpy().tolist()


_EIG = {}


def _eig_engine(H, C):
    if H == 1024:
        return _case(1024)
    if (H, C) not in _EIG:
        hard = design_hard(H, C, 150, seed=H + C, many=(33, 70) if H >= 70 else (), twice=True)
        _ENGINES[("eig", H, C)] = _selector(slab_from_hard(hard, C, seed=C, twice=True))
        _EIG[(H, C)] = _ENGINES[("eig", H, C)].engine
    return _EIG[(H, C)]


def g8_kc(C):
    return 4 if C <= 32 else 8 if C <= 64 else 13 if C <= 104 else 16


def kc_of(C):
    return 1 if C <= 32 else 2 if C <= 64 else 4 if C <= 128 else 0


@pytest.mark.gpu
@pytest.mark.parametrize("H,C", [(12, c) for c in (2, 32, 33, 64, 65, 104, 105, 128, 129, 300, 1000)]
                         + [(80, 100), (80, 300), (1024, 100)])
def test_eig_assembly_and_records_match_a_host_evaluation(H, C):
    """eig against eig64 on the kernel's own gains and U on every assembly path -- the 8-lane kernel with the ELL copy
    (every KC8 bucket edge), without it (raw ABI), k_gain_eig<KC> for KC = 1, 2, 4 (max_entries = -1) and KC = 0
    (C > 128), and items with 33 and 70 distinct classes (the entry loop goes round two and three times) -- and the
    merged records equal to a host evaluation on the kernel's eig vector, exactly.  Every item has an identical twin,
    so the best candidate is an exact tie that only the first-index rule decides."""
    e = _eig_engine(H, C)
    assert e.C == C and e.H == H
    with e._on():
        e.scored = False
        e._score()
    _flags_clear(e)
    nent = np.diff(e.ent_off.cpu().numpy())
    assert e.max_entries == nent.max()
    if H >= 70:
        assert (nent == 33).any() and (nent == 70).any() and e.ell_k == 0
    gain = e.gain.cpu().numpy()
    variants = []
    if C <= 128 and e.max_entries <= 32:
        assert e.ell_k == (e.max_entries + 3) // 4 * 4
        variants += [(f"g8<{g8_kc(C)}> ell", e.max_entries, e.ell_row, e.ell_cls, e.ell_k),
                     (f"g8<{g8_kc(C)}> no ell", e.max_entries, None, None, 0)]
    variants.append((f"k_gain_eig<{kc_of(C)}>", -1 if C <= 128 else e.max_entries, None, None, 0))
    ref, bound = eig64(e, gain)
    # label the twins of the three lowest-scored candidate pairs and one unanimous item (never the best pair)
    dis = e.disagree.cpu().numpy().astype(bool)
    order = np.argsort(ref[0::2] + np.where(dis[0::2], 0, np.inf))
    lab = [2 * int(i) + 1 for i in order[:3]] + [2 * int(np.flatnonzero(~dis[0::2])[0])]
    e.labeled[torch.tensor(lab, device=e.dev)] = 1
    labeled = e.labeled.cpu().numpy().astype(bool)
    for name, me, er, ec, ek in variants:
        eig, rec = launch_eig(e, me, er, ec, ek)
        assert np.isfinite(eig).all()
        ratio = float((np.abs(eig - ref) / bound).max())
        _report("eig", f"C={C} H={H} {name}", float(np.abs(eig - ref).max()), float(bound.max()))
        assert ratio <= 1, ratio
        assert rec == host_record(eig, labeled, dis), name
        assert rec[0] == rec[5] and rec[1] % 2 == 0          # the best candidate is tied with its twin
        assert rec != host_record(eig, labeled, dis, last=True)
    # negative control: g0 of the two most frequent classes swapped in the model
    cnt = np.bincount(e.ent_cls.cpu().numpy().astype(np.int64) & 0xFFFF, minlength=C)
    top2 = tuple(int(c) for c in np.argsort(-cnt)[:2])
    bad, _ = eig64(e, gain, swap=top2)
    assert (np.abs(eig - bad) / bound).max() > 1


# ------------------------------------------------------------------------------------------------------------------
# stage 5: mixture
# ------------------------------------------------------------------------------------------------------------------
def check_mixture(e, label, stale=None):
    """k_step_mixture into poisoned outputs: pi_hat = fp32(pisum / total) exactly, m0 = sum_c pi_hat PB within the
    fp32 bound of four interleaved FMA chains of non-negative terms ((C / 4 + 3) u m0), zero padding, H_before within
    the bound of its fp32 entropy terms, and best_model the first index of the largest m0."""
    with e._on():
        e.m0.fill_(NAN)
        e.hb.fill_(NAN)
        e.pi_hat.fill_(NAN)
        e.best_model.fill_(-7)
        e._mixture()
    _flags_clear(e)
    H, C = e.H, e.C
    ps = e.pisum.cpu().numpy()
    pi = e.pi_hat.cpu().numpy()
    assert np.array_equal(pi, (ps.astype(np.float64) / float(ps.sum())).astype(np.float32))
    PB = e.PB.cpu().numpy().astype(np.float64)[:, :H]
    m0 = e.m0.cpu().numpy()
    assert np.isfinite(m0).all() and (m0[H:] == 0).all()
    mm = pi.astype(np.float64) @ PB
    tol = (C / 4 + 3) * U32 * mm + 1e-45
    err = np.abs(m0[:H] - mm)
    _report("mixture", f"{label} m0 (ulp)", float((err / (U32 * mm)).max()), C / 4 + 3)
    assert (err <= tol).all()
    m = m0[:H].astype(np.float64)
    hb, hb_tol = ent64(m).sum(), ent_bound(m).sum() + 17 * U32 * ent64(m).sum()
    _report("mixture", f"{label} H_before", abs(float(e.hb.item()) - hb), hb_tol)
    assert abs(float(e.hb.item()) - hb) <= hb_tol
    assert int(e.best_model.item()) == int(np.argmax(m0[:H]))
    if stale is not None:
        old = stale[0].astype(np.float64) @ stale[1].astype(np.float64)[:, :H]
        assert (np.abs(m0[:H] - old) > tol).any()
    return m0


@pytest.mark.gpu
@pytest.mark.parametrize("H", [300, 1024])
def test_mixture_matches_the_fp64_model(H):
    check_mixture(_case(H), f"H={H}")


@pytest.mark.gpu
def test_mixture_breaks_an_exact_tie_by_the_first_index():
    """Models 3 and 4 are identical and always right: their PB columns, hence m0, are the same bits and the largest,
    and the best model is 3 -- after construction and after a label.  The m0 of the step before the label does not
    pass the comparison (negative control)."""
    H, C, N = 12, 10, 400
    rng = np.random.default_rng(4)
    y = rng.integers(0, C, N)
    hard = np.where(rng.random((N, H)) < 0.6, y[:, None], (y[:, None] + rng.integers(1, 4, (N, H))) % C)
    hard[:, 3] = hard[:, 4] = y
    preds = slab_from_hard(hard, C, seed=4)
    preds[4] = preds[3]
    sel = _selector(preds)
    e = sel.engine
    m0 = check_mixture(e, "tie")
    assert m0[3] == m0[4] == m0[:H].max() and int(e.best_model.item()) == 3
    prev = (e.pi_hat.cpu().numpy(), e.PB.cpu().numpy())
    i = int(np.flatnonzero((hard != hard[:, :1]).any(1))[0])
    sel.add_label(i, int(y[i]), 0.0)
    torch.cuda.synchronize()
    m0 = check_mixture(e, "tie, one label later", stale=prev)
    assert m0[3] == m0[4] == m0[:H].max() and int(e.best_model.item()) == 3
    sel.close()


# ------------------------------------------------------------------------------------------------------------------
# stage 6: incremental state
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("tc", [True, False])
def test_incremental_refresh_leaves_what_a_full_rebuild_writes(tc):
    """After labels of a class with the most row tiles and of classes with fewer (whose ``sel`` launches end with
    CTAs that exit early), the row cache is bit-identical to a full refill and the tables to a full rebuild from the
    current D; the padded model columns of G0T / G1T / PB / the limbs stay zero.  The cache from before the last
    label differs from the refill (negative control)."""
    H, C = 200, 5
    hard = design_hard(H, C, 24, seed=21, heavy={0: 300})
    sel = _selector(slab_from_hard(hard, C, seed=21), tc=tc)
    e = sel.engine
    assert e.use_tc == tc and e.Hp == 224 and e.mode == "incremental"
    ntile = np.diff(e.tile_off_host)
    assert ntile[0] == e.max_cls_tiles > ntile[1:].max()
    check_padding(e)
    sel.get_next_item_to_label()                                   # fills the row cache
    steps = [(0, 0), (1, 1), (2, 0), (3, 2), (4, 1)]               # (item, class)
    assert {t for _, t in steps} >= {0, 1} and all(hard[i].min() != hard[i].max() for i, _ in steps)
    for k, (i, t) in enumerate(steps):
        if k == len(steps) - 1:
            torch.cuda.synchronize()
            before = e.ph_cache.clone()
        sel.add_label(i, t, 0.0)
    torch.cuda.synchronize()
    check_padding(e)
    t = fresh_tables(H, C, tc)
    launch_tables(e.D, H, C, 0, C, t)
    for k in t:
        assert same_bits(t[k], getattr(e, k)), k
    ph, _ = launch_rows(e, tc, gains=False)
    assert same_bits(ph, e.ph_cache)
    assert not same_bits(before, ph)
    sel.close()
