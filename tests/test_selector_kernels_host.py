"""Host models of the competing selectors' kernels (csrc/baselines.cu, csrc/bl_ref.cu) and the CPU tests that tie each
model to the reference's own formulas and goldens, so that tests/test_selector_kernels.py compares every kernel with
something trusted.

  static     k_static_scores         ActiveTesting / VMA scores: exact integer sums, one fp32 rounding     bit for bit
  entropy    k_mp_entropy            the grouped closed form of DESIGN.md §5b in long double                 <= 1/2 ulp + fp64 bound
  posterior  k_bl_step (ModelPicker) fp32 products, the fixed-order fp64 sum, one rounding, fp32 division  bit for bit
  lure       k_bl_step / bl_best_ref fl(fma(N - m, s2, s1) / m) and the exact rational LURE of get_vs()
  draw       weighted_draw_xchg      random.choices on the kernel's fp32-normalised weights

Run with ``-s`` to see the worst error of every comparison against its bound."""
import bisect
import itertools
import math
import random
from fractions import Fraction

import numpy as np
import pytest
import torch

from helpers import GOLDEN, synth

U32 = 2.0 ** -24                      # fp32 unit roundoff
U64 = 2.0 ** -53                      # fp64 unit roundoff
LD = np.longdouble


def report(stage, label, err, tol):
    print(f"[selector] {stage:<9} {label:<52} worst {err:.3e}   bound {tol:.1e}")


# ------------------------------------------------------------------------------------------------------------------
# ActiveTesting / VMA static scores (k_static_scores)
# ------------------------------------------------------------------------------------------------------------------
def model_losses(g, H):
    """l = fp32(1 - fp32(e / H)) for the gathered ensemble sums g = ens[n, hard[n, h]] (any shape, fp32)."""
    g = np.asarray(g, np.float32)
    return np.float32(1.0) - g / np.float32(H)


def static_exact(g, H):
    """(at, vma) fp32 of every item from g [N][H] = ens[n, hard[n, h]].  Every loss is a multiple of 2^-24 (1 - x with
    x in [0.5, 1] is exact, anything else rounds into [0.5, 1]), and a score is at most H·H/4 such units, so the fp64
    sums of the kernel are exact in any order: the score is the exact integer sum times 2^-24, rounded once to fp32.
    VMA over models equals the grouped sum over classes (models in one group add |l - l| = 0); with the losses sorted,
    sum_{h<h'} |l_h - l_h'| = sum_k l_(k) (2k - H + 1)."""
    l = model_losses(g, H).astype(np.float64)
    li = l * 2.0 ** 24
    assert np.array_equal(li, np.round(li)), "a loss is not a multiple of 2^-24"
    li = li.astype(np.int64)
    at = li.sum(1)
    w = 2 * np.arange(H, dtype=np.int64) - H + 1
    vma = (np.sort(li, axis=1) * w).sum(1)
    return ((at.astype(np.float64) * 2.0 ** -24).astype(np.float32),
            (vma.astype(np.float64) * 2.0 ** -24).astype(np.float32))


def warp_butterfly(part):
    """warp_sum over 32 lane values: v_lane += v_(lane ^ o) for o = 16, 8, 4, 2, 1 (lane 0's result)."""
    v = [float(x) for x in part]
    for o in (16, 8, 4, 2, 1):
        v = [v[i] + v[i ^ o] for i in range(32)]
    return v[0]


def static_ordered(hard_row, ens_row, H):
    """k_static_scores for one item, step by step: the groups in order of their lowest model, AT as the running fp64 sum
    of m_k·l_k, VMA as lane partials (i = lane mod 32, j > i ascending) then the butterfly; one fp32 rounding each."""
    order = list(dict.fromkeys(int(c) for c in hard_row))
    m = [int((hard_row == c).sum()) for c in order]
    l = [float(model_losses(ens_row[c], H)) for c in order]
    at = 0.0
    for mk, lk in zip(m, l):
        at += float(mk) * lk
    part = [0.0] * 32
    K = len(order)
    for i in range(K):
        for j in range(i + 1, K):
            part[i % 32] += float(m[i]) * float(m[j]) * abs(l[i] - l[j])
    return np.float32(at), np.float32(warp_butterfly(part))


def at_literal(p):
    """activetesting.py's acquisition before normalisation: sum_h (1 - mean_h p[h, n, argmax_c p[h, n]]), fp64."""
    p = np.asarray(p, np.float64)
    H, N, _ = p.shape
    ens = p.mean(0)
    return (1.0 - ens[np.arange(N)[None], p.argmax(2)]).sum(0)


def vma_literal(p):
    """vma.py's pairwise sum_{h < h'} |l_h - l_h'| over the models, fp64."""
    p = np.asarray(p, np.float64)
    H, N, _ = p.shape
    l = 1.0 - p.mean(0)[np.arange(N)[None], p.argmax(2)]
    iu = np.triu_indices(H, 1)
    return np.abs(l[:, None] - l[None, :])[iu].sum(0)


def scan_gather(p32):
    """(hard [N][H], g [N][H]) of an fp32 slab as the scan leaves them: first arg-max, E summed in model order (fp32)."""
    H = p32.shape[0]
    E = np.zeros(p32.shape[1:], np.float32)
    for h in range(H):
        E += p32[h]
    hard = p32.argmax(2).T
    return hard, E[np.arange(hard.shape[0])[:, None], hard]


def crafted_rows(H, C, N, rng):
    """hard [N][H] int64 whose first rows have K = 1, 2, 31, 32, 33 and min(H, C) distinct classes (those that fit),
    groups of very unequal size (K - 1 single models and one group of the rest, the big group's lowest model placed at
    random), then random rows; the classes are random ids in [0, C)."""
    hard = rng.integers(0, C, (N, H))
    ks = [k for k in dict.fromkeys((1, 2, 31, 32, 33, min(H, C))) if k <= min(H, C)]
    r = 0
    for k in ks:
        for _ in range(3):
            if r >= N:
                break
            cls = rng.choice(C, size=k, replace=False)
            row = np.full(H, cls[0])
            pos = rng.permutation(H)[: k - 1]
            row[pos] = cls[1:]
            hard[r] = row
            r += 1
    if C > 1 and r < N:                                 # few distinct classes: the synthetic tasks' common case
        hard[r:min(N, r + 32)] = rng.integers(0, min(C, 3), (min(N, r + 32) - r, H))
    return hard, ks


def test_static_models_agree_with_each_other_and_the_literal_formulas():
    rng = np.random.default_rng(0)
    worst = [0.0, 0.0]
    for H, C in ((1, 2), (5, 3), (33, 100), (70, 40), (257, 300)):
        hard, _ = crafted_rows(H, C, 40, rng)
        ens = (rng.random((40, C)) * H).astype(np.float32)
        ens[0, hard[0, 0]] = np.float32(H)              # l = 0
        ens[1, hard[1, 0]] = 0.0                        # l = 1
        g = ens[np.arange(40)[:, None], hard]
        at, vma = static_exact(g, H)
        for n in range(40):
            a, v = static_ordered(hard[n], ens[n], H)
            assert a.view(np.uint32) == at[n].view(np.uint32) and v.view(np.uint32) == vma[n].view(np.uint32), (H, C, n)
        # the model over models: sum_h l_h and sum_{h<h'} |l_h - l_h'| in exact arithmetic
        l = model_losses(g, H).astype(np.float64)
        for n in range(40):
            ex_at = math.fsum(l[n])
            ex_v = math.fsum(abs(l[n, i] - l[n, j]) for i, j in itertools.combinations(range(H), 2))
            assert at[n] == np.float32(ex_at) and vma[n] == np.float32(ex_v)
    # against activetesting.py / vma.py on slabs: the kernel's losses round e / H and 1 - x to fp32, the reference's
    # fp32 mean rounds similarly; both are within (H + 2) fp32 roundings of the fp64 literal value per loss
    for H, N, C, seed in ((6, 200, 5, 1), (24, 150, 100, 2)):
        p, _ = synth(H, N, C, seed)
        p = p.numpy()
        hard, g = scan_gather(p)
        at, vma = static_exact(g, H)
        lat, lvma = at_literal(p), vma_literal(p)
        tol_at = (H + 3) * U32 * H
        tol_v = (H + 3) * U32 * H * H
        worst[0] = max(worst[0], float(np.abs(at - lat).max()))
        worst[1] = max(worst[1], float(np.abs(vma - lvma).max()))
        assert np.abs(at - lat).max() <= tol_at and np.abs(vma - lvma).max() <= tol_v
    report("static", "model vs activetesting.py / vma.py (abs)", max(worst), 1e-4)


@pytest.mark.parametrize("name", ["baseline_activetesting_h12_n500_c6", "baseline_activetesting_h24_n400_c100",
                                  "baseline_vma_h12_n500_c6", "baseline_vma_h24_n400_c100",
                                  "baseline_activetesting_h256_n1500_c100", "baseline_vma_h256_n1500_c100"])
def test_static_model_reproduces_the_goldens_scores(name):
    """The bit model on the slab synth rebuilds gives the reference's fp32 scores within the reference's own fp32
    error: its mean over H models (H roundings per loss) and its fp32 sum over H (or H(H-1)/2 pair) terms."""
    z = np.load(f"{GOLDEN}/{name}.npz")
    H, N, C = int(z["H"]), int(z["N"]), int(z["C"])
    p, _ = synth(H, N, C, int(z["data_seed"]))
    hard, g = scan_gather(p.numpy())
    at, vma = static_exact(g, H)
    got = vma if "_vma_" in name else at
    ref = z["score"].astype(np.float64)
    terms = H * (H - 1) / 2 if "_vma_" in name else H
    tol = 2 * (H + terms) * U32 * np.maximum(np.abs(ref), 1.0)
    err = np.abs(got - ref)
    report("static", f"{name} score", float((err / tol).max()) * tol.max(), float(tol.max()))
    assert (err <= tol).all()


# ------------------------------------------------------------------------------------------------------------------
# ModelPicker entropy (k_mp_entropy)
# ------------------------------------------------------------------------------------------------------------------
def gamma_of(eps):
    """gamma as the kernels receive it: (1 - eps) / eps rounded to fp32 (modelpicker.py:78 multiplies in fp32)."""
    return float(np.float32((1.0 - eps) / eps))


def entropy_ld(hard_row, post32, C, gamma):
    """DESIGN.md §5b's grouped closed form in long double -> (value, K): p_h the fp32 posterior widened exactly,
    0·log 0 = 0."""
    p = np.asarray(post32, np.float32).astype(LD)
    pl = np.where(p > 0, p * np.log2(np.where(p > 0, p, LD(1))), LD(0))
    S, B = p.sum(), pl.sum()
    gm = LD(gamma)
    gm1, glg = gm - 1, gm * np.log2(gm)
    cls, inv = np.unique(np.asarray(hard_row), return_inverse=True)
    a = np.zeros(len(cls), LD)
    q = np.zeros(len(cls), LD)
    np.add.at(a, inv, p)
    np.add.at(q, inv, pl)
    norm = S + gm1 * a
    acc = (np.log2(norm) - (B + gm1 * q + glg * a) / norm).sum()
    K = len(cls)
    return (acc + (C - K) * (np.log2(S) - B / S)) / C, K


def entropy_fp64_bound(post32, H, K, gamma):
    """|fp64 evaluation - exact| for k_mp_entropy.  S, B and each group's a, q are fp64 sums of at most H terms of one
    sign (relative error H·u each, p log2 p adding 2 roundings and CUDA's 1-ulp log2); each of the K + 2 terms (K groups,
    H_none and its (C - K) multiple) takes <= 10 more roundings of quantities bounded by
    T = |log2 S| + log2 max(gamma, 1) + 1 + (|B| + gamma |log2 gamma| S) / S, and the terms enter a running sum:
    |err| <= (2H + 12 (K + 2))·u·T."""
    p = np.asarray(post32, np.float64)
    S = p.sum()
    B = np.abs(np.where(p > 0, p * np.log2(np.where(p > 0, p, 1.0)), 0.0)).sum()
    T = abs(math.log2(S)) + math.log2(max(gamma, 1.0)) + 1.0 + (B + gamma * abs(math.log2(gamma)) * S) / S
    return (2 * H + 12 * (K + 2)) * U64 * T


def entropy_tol(value, post32, H, K, gamma):
    """Half an fp32 ulp of the value (the one rounding) plus the fp64 evaluation bound."""
    v = abs(float(value))
    half_ulp = 0.5 * (np.spacing(np.float32(v)) if v > 0 else np.float32(2.0 ** -149))
    return float(half_ulp) + entropy_fp64_bound(post32, H, K, gamma)


def clamped_loop_entropy(hard_row, post32, C, gamma):
    """modelpicker.py's per-class loop for one item in fp64, with its clamp at 1e-12."""
    post = np.asarray(post32, np.float64)
    out = 0.0
    for c in range(C):
        w = post * gamma ** (np.asarray(hard_row) == c).astype(np.float64)
        pc = np.maximum(w / w.sum(), 1e-12)
        out += -(pc * np.log2(pc)).sum() / C
    return out


def posteriors(H, rng):
    """Uniform, peaked, and with fp32-subnormal and exactly-zero entries, each normalised in fp32."""
    out = {"uniform": np.full(H, np.float32(1.0 / H), np.float32)}
    pk = rng.dirichlet(np.full(H, 0.05)).astype(np.float32)
    out["peaked"] = pk / pk.sum(dtype=np.float32)
    sub = rng.dirichlet(np.ones(H)).astype(np.float32)
    if H > 1:
        k = max(1, H // 3)
        idx = rng.permutation(H)[: 2 * k]
        sub[idx[:k]] = (rng.integers(1, 1 << 23, k) * 2.0 ** -149).astype(np.float32)    # subnormal
        sub[idx[k:2 * k]] = 0.0
    out["subnormal"] = sub
    return out


def test_entropy_model_matches_the_clamped_loop():
    rng = np.random.default_rng(4)
    worst = 0.0
    for H, C in ((1, 2), (5, 3), (33, 100), (256, 100), (64, 10)):
        for eps in (0.35, 0.46, 0.49, 0.5):
            gm = gamma_of(eps)
            for kind, post in posteriors(H, rng).items():
                for _ in range(3):
                    row = rng.integers(0, min(C, 11), H)
                    v, K = entropy_ld(row, post, C, gm)
                    ref = clamped_loop_entropy(row, post, C, gm)
                    err = abs(float(v) - ref)
                    worst = max(worst, err)
                    assert err <= H * 4e-11 + 1e-12, (H, C, eps, kind, err)
    report("entropy", "long double model vs clamped loop (fp64)", worst, 1024 * 4e-11)
    # gamma = 1 (eps = 0.5): a label changes nothing, so every item scores the entropy of the posterior
    post = posteriors(40, rng)["peaked"]
    v, _ = entropy_ld(rng.integers(0, 5, 40), post, 7, gamma_of(0.5))
    p = post.astype(LD)
    S = p.sum()
    assert abs(v - (np.log2(S) - (p[p > 0] * np.log2(p[p > 0])).sum() / S)) < 1e-15


def test_entropy_model_reproduces_the_goldens_entropies():
    """On the ModelPicker goldens' posteriors (the reference's own fp32 state at every step) the model gives the
    reference's entropies within the reference's fp32 running sum over C classes."""
    for name in ("baseline_model_picker_h12_n500_c6", "baseline_model_picker_h24_n400_c100"):
        z = np.load(f"{GOLDEN}/{name}.npz")
        H, N, C = int(z["H"]), int(z["N"]), int(z["C"])
        p, _ = synth(H, N, C, int(z["data_seed"]))
        hard = p.numpy().argmax(2).T
        gm = gamma_of(0.46)
        worst, tol = 0.0, C * 2 * U32 * math.log2(max(H, 2)) + 2e-6
        for s in range(1, int(z["steps"]), 7):
            post = z["posterior"][s - 1]
            ent = z["ent"][s]
            for n in np.nonzero(np.isfinite(ent))[0][:25]:
                v, _ = entropy_ld(hard[n], post, C, gm)
                worst = max(worst, abs(float(v) - float(ent[n])))
        report("entropy", f"{name} ent", worst, tol)
        assert worst <= tol


# ------------------------------------------------------------------------------------------------------------------
# ModelPicker posterior (k_bl_step)
# ------------------------------------------------------------------------------------------------------------------
def posterior_step(post32, agree, gamma32, threads=256):
    """k_bl_step's update: p_h = fp32(post_h · gamma) where the model agrees with the label; thread t sums
    h = t, t + 256, ... in fp64, each warp's 32 partials by the xor butterfly, the 8 warps in order; the sum rounded
    once to fp32; post_h = fp32(p_h / sum)."""
    post32 = np.asarray(post32, np.float32)
    p = np.where(agree, post32 * np.float32(gamma32), post32).astype(np.float32)
    H = p.size
    rows = -(-H // threads)
    pad = np.zeros(rows * threads)
    pad[:H] = p
    pad = pad.reshape(rows, threads)
    part = pad[0].copy()
    for r in range(1, rows):
        part = part + pad[r]
    s = 0.0
    for w in range(threads // 32):
        s += warp_butterfly(part[32 * w:32 * w + 32])
    return (p / np.float32(s)).astype(np.float32)


def torch_posterior_step(post32, agree, gamma):
    """modelpicker.py's update in torch (fp32 sum)."""
    post = torch.from_numpy(np.asarray(post32, np.float32))
    nxt = post * (gamma ** torch.from_numpy(np.asarray(agree)).float())
    return (nxt / nxt.sum()).numpy()


def ulps32(a, b):
    a = np.asarray(a, np.float32).view(np.int32).astype(np.int64)
    b = np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


@pytest.mark.parametrize("name", ["baseline_model_picker_h12_n500_c6", "baseline_model_picker_h24_n400_c100",
                                  "baseline_model_picker_h256_n1500_c100"])
def test_posterior_model_reproduces_the_goldens_posterior(name):
    """Replayed along the reference's picks, the fixed-order update stays within a few ulps of the goldens' torch
    posterior at every step, and of torch's own update applied to the same state."""
    z = np.load(f"{GOLDEN}/{name}.npz")
    H, N, C = int(z["H"]), int(z["N"]), int(z["C"])
    p, labels = synth(H, N, C, int(z["data_seed"]))
    hard = p.numpy().argmax(2).T
    gm = (1.0 - 0.46) / 0.46
    post = np.full(H, np.float32(1.0 / H), np.float32)
    worst_g = worst_t = 0
    for s, idx in enumerate(z["idx"]):
        agree = hard[idx] == labels.numpy()[idx]
        t = torch_posterior_step(post, agree, gm)
        post = posterior_step(post, agree, np.float32(gm))
        worst_t = max(worst_t, int(ulps32(post, t).max()))
        worst_g = max(worst_g, int(ulps32(post, z["posterior"][s]).max()))
    report("posterior", f"{name} (ulps vs golden / torch step)", max(worst_g, worst_t), 8 + s // 4)
    assert worst_t <= 4 and worst_g <= 8 + s // 4


def test_posterior_model_matches_torch_on_long_runs():
    rng = np.random.default_rng(5)
    for H in (1, 7, 256, 257, 1000, 1024):
        post = np.full(H, np.float32(1.0 / H), np.float32)
        acc = rng.uniform(0.3, 0.95, H)
        worst = 0
        for _ in range(300):
            agree = rng.random(H) < acc
            t = torch_posterior_step(post, agree, gamma_of(0.35))
            post = posterior_step(post, agree, gamma_of(0.35))
            worst = max(worst, int(ulps32(post, t).max()))
            assert np.all(post >= 0) and abs(float(post.astype(np.float64).sum()) - 1.0) < H * 1e-6
        report("posterior", f"H={H} one step vs torch (ulps)", worst, 4)
        assert worst <= 4


# ------------------------------------------------------------------------------------------------------------------
# LURE (k_bl_step, k_bl_best_ref)
# ------------------------------------------------------------------------------------------------------------------
def lure_t(Ng, m, q):
    """S2's increment of label m (1-based) with selection probability q, as k_bl_step computes it in fp64."""
    am = 1.0 / ((Ng - m + 1.0) * q) - 1.0
    return am / (Ng - m) if Ng - m > 0.0 else 0.0


def fma(a, b, c):
    """Correctly rounded a·b + c in fp64."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def lure_risk(s1, s2, Ng, m):
    """bl_lure_risk: fl(fma(Ng - m, s2, s1) / m)."""
    return fma(Ng - m, s2, s1) / m


def lure_sums(Ng, qs, L):
    """The loop's running sums s1, s2 [H] after the labels with probabilities qs and losses L [M][H], in label order."""
    H = L.shape[1]
    s1, s2 = np.zeros(H), np.zeros(H)
    for m, (q, row) in enumerate(zip(qs, L), start=1):
        t = lure_t(float(Ng), float(m), float(q))
        s1 = s1 + np.where(row, 1.0, 0.0)
        s2 = s2 + np.where(row, t, 0.0)
    return s1, s2


def lure_exact(N, qs, L):
    """activetesting.py's LURE risk per model as an exact rational: mean_m v_m L_mh with
    v_m = 1 + (N - M)/(N - m) · (1/((N - m + 1) q_m) - 1).  At M = N the factor (N - M)/(N - m) is 0/0 for m = N, where
    get_vs divides by zero; the loop takes v_m = 1 there (the factor is 0 for every other m), the plain mean."""
    M = len(qs)
    vs = []
    for m, q in enumerate(qs, start=1):
        f = Fraction(N - M, N - m) if m < N else Fraction(0)
        vs.append(1 + f * (1 / ((N - m + 1) * Fraction(float(q))) - 1))
    return [sum((vs[m] for m in np.nonzero(L[:, h])[0]), Fraction(0)) / M for h in range(L.shape[1])]


def lure_bound(N, qs, s1, s2):
    """|fl risk - exact| for the loop's fp64 evaluation.  Each increment t_m takes 4 roundings: the product
    (N - m + 1)·q (exact below 2^53), 1/x, -1 (absolute error u·|1/x|) and / (N - m); S2 then adds at most M of them
    (a running sum: M·u·sum|t|); the risk takes the fma and the division: 2u·|risk| more."""
    M = len(qs)
    per = [(abs(1.0 / ((N - m + 1) * q)) + abs(lure_t(N, m, q)) * (N - m)) * 3 * U64 / max(N - m, 1)
           for m, q in enumerate(qs, start=1)]
    e_t = sum(per)
    sum_t = sum(abs(lure_t(N, m, q)) for m, q in enumerate(qs, start=1))
    e_s2 = e_t + M * U64 * sum_t
    risk = np.abs(s1 + (N - M) * s2) / M
    return ((N - M) * e_s2) / M + 3 * U64 * risk


def test_lure_models_reproduce_the_goldens_lure():
    """The running sums and the rational model along the goldens' picks and q give the reference's fp32 LURE risks at
    every step (torch's fp32 products and mean: within 1e-6 absolute at these sizes, as test_baselines.py)."""
    for name in ("baseline_activetesting_h12_n500_c6", "baseline_activetesting_h24_n400_c100",
                 "baseline_vma_h12_n500_c6", "baseline_vma_h24_n400_c100"):
        z = np.load(f"{GOLDEN}/{name}.npz")
        H, N, C = int(z["H"]), int(z["N"]), int(z["C"])
        p, labels = synth(H, N, C, int(z["data_seed"]))
        hard = p.numpy().argmax(2).T
        L = hard[z["idx"]] != labels.numpy()[z["idx"]][:, None]
        worst = 0.0
        for s in range(len(z["idx"])):
            qs = list(z["q"][: s + 1])
            ex = np.array([float(v) for v in lure_exact(N, qs, L[: s + 1])])
            s1, s2 = lure_sums(N, qs, L[: s + 1])
            fl = np.array([lure_risk(a, b, float(N), float(s + 1)) for a, b in zip(s1, s2)])
            bound = lure_bound(N, qs, s1, s2)
            assert (np.abs(fl - ex) <= bound + 1e-300).all(), (name, s)
            worst = max(worst, float(np.abs(ex - z["lure"][s]).max()))
        report("lure", f"{name} exact vs golden", worst, 1e-6)
        assert worst <= 1e-6


def test_lure_models_match_the_weighted_sum_identity():
    """The identity of test_baselines_loop_host.py::test_lure_identity_equals_the_weighted_sum, exactly: the rational
    model equals (S1 + (N - M) S2) / M in rationals, and the fp64 sums are within lure_bound of it; at M = N the risk
    is the plain mean."""
    rng = np.random.default_rng(3)
    for N, M, H in ((500, 40, 12), (10_000, 300, 16), (50, 49, 5), (60, 60, 6)):
        qs = [float(np.float32(x)) for x in rng.uniform(1e-4, 0.05, M)]
        L = rng.integers(0, 2, (M, H)).astype(bool)
        ex = lure_exact(N, qs, L)
        def t_exact(m):                                 # a_m / (N - m), m 1-based; 0 at m = N
            return (1 / ((N - m + 1) * Fraction(qs[m - 1])) - 1) / (N - m) if m < N else Fraction(0)
        S2 = [sum((t_exact(i + 1) for i in np.nonzero(L[:, h])[0]), Fraction(0)) for h in range(H)]
        for h in range(H):
            assert (int(L[:, h].sum()) + (N - M) * S2[h]) / M == ex[h]
        s1, s2 = lure_sums(N, qs, L)
        fl = np.array([lure_risk(a, b, float(N), float(M)) for a, b in zip(s1, s2)])
        err = np.abs(fl - np.array([float(v) for v in ex]))
        bound = lure_bound(N, qs, s1, s2)
        report("lure", f"N={N} M={M} fp64 sums vs rational", float(err.max()), float(bound.max()))
        assert (err <= bound).all()
        if M == N:
            assert all(ex[h] == Fraction(int(L[:, h].sum()), M) for h in range(H))
            assert np.array_equal(fl, s1 / M)


def test_lure_fma_model_differs_from_the_uncontracted_one():
    """The tie model is sharp: a plain multiply-then-add rounds some of these risks differently from the fma."""
    rng = np.random.default_rng(8)
    diff = 0
    for _ in range(2000):
        s1 = float(rng.integers(0, 50))
        s2 = float(rng.uniform(-0.01, 0.05))
        Ng, m = 5000.0, float(rng.integers(1, 4999))
        diff += lure_risk(s1, s2, Ng, m) != (s1 + (Ng - m) * s2) / m
    assert diff > 0


# ------------------------------------------------------------------------------------------------------------------
# weighted draw (random.choices)
# ------------------------------------------------------------------------------------------------------------------
def normalised(w, labeled, total):
    """The kernel's fp32 weights of the unlabeled items: fp32(w / fp32(total)), in index order."""
    unl = np.nonzero(~np.asarray(labeled, bool))[0]
    return unl, (np.asarray(w, np.float32)[unl] / np.float32(total)).astype(np.float32)


def choices_draw(wn, u):
    """random.choices(population, weights=wn)[0] with random() = u, literally: the position among the unlabeled items
    and the cumulative weights."""
    cum = list(itertools.accumulate(float(x) for x in wn))
    return bisect.bisect(cum, u * (cum[-1] + 0.0), 0, len(cum) - 1), cum


def boundary_distance(cum, pos, u):
    """Relative distance of the target u·total from the nearer end of the chosen item's interval."""
    total = cum[-1]
    t = u * total
    lo = cum[pos - 1] if pos > 0 else 0.0
    return min(abs(t - lo), abs(cum[pos] - t)) / total if total > 0 else 0.0


def test_draw_model_is_random_choices():
    rng = np.random.default_rng(9)
    random.seed(17)
    for n in (1, 2, 7, 300, 5000):
        for trial in range(30):
            w = (rng.random(n) ** 3).astype(np.float32)
            w[rng.random(n) < 0.2] = 0
            if trial % 3 == 0 and n > 3:
                w[-3:] = 0                                  # zero weights at the end: bisect's hi fallback
            labeled = rng.random(n) < 0.2
            labeled[-1] = False
            if w[~labeled].sum() == 0:
                w[-1] = 1.0
            total = float(w[~labeled].astype(np.float64).sum())
            unl, wn = normalised(w, labeled, total)
            state = random.getstate()
            ref = random.choices(list(unl), weights=[float(x) for x in wn])[0]
            random.setstate(state)
            pos, _ = choices_draw(wn, random.random())
            assert unl[pos] == ref, (n, trial)
    # the largest random() still picks the last item of positive weight, not the zero-weight tail
    pos, _ = choices_draw(np.array([0.25, 0.75, 0.0, 0.0], np.float32), math.nextafter(1.0, 0.0))
    assert pos == 1
