"""CPU models of the baseline kernels (csrc/baselines.cu) against the literal formulas of the selectors they replace,
and the ``coda.baselines`` shim without a reference checkout."""
import bisect
import itertools
import os
import random
import subprocess
import sys

import numpy as np

from helpers import ROOT


def literal_mp_entropy(hard_row, post, C, gamma):
    """modelpicker.py:74-86 for one item, in fp64: the per-class loop with the 1e-12 clamp."""
    out = 0.0
    for c in range(C):
        w = post * gamma ** (hard_row == c).astype(np.float64)
        p = np.maximum(w / w.sum(), 1e-12)
        out += -(p * np.log2(p)).sum() / C
    return out


def xlog2x(p):
    return np.where(p > 0, p * np.log2(np.where(p > 0, p, 1.0)), 0.0)


def grouped_mp_entropy(hard_row, post, C, gamma):
    """What k_mp_entropy computes: one term per distinct predicted class, groups in order of their lowest model."""
    S, B = post.sum(), xlog2x(post).sum()
    pl = xlog2x(post)
    acc, K = 0.0, 0
    for c in dict.fromkeys(hard_row.tolist()):            # first-occurrence order == lowest model index
        z = hard_row == c
        a, q = post[z].sum(), pl[z].sum()
        norm = S + (gamma - 1) * a
        acc += np.log2(norm) - (B + (gamma - 1) * q + gamma * np.log2(gamma) * a) / norm
        K += 1
    return (acc + (C - K) * (np.log2(S) - B / S)) / C


def test_grouped_modelpicker_entropy_equals_the_per_class_loop():
    rng = np.random.default_rng(0)
    worst = 0.0
    for H, C in ((5, 3), (24, 100), (256, 100), (64, 10)):
        gamma = (1 - 0.46) / 0.46
        for trial in range(20):
            post = rng.dirichlet(np.ones(H) * (0.05 if trial % 2 else 5.0))
            if trial % 4 == 1:
                post[rng.integers(0, H, size=max(1, H // 5))] = 0.0          # underflowed posteriors: 0 log 0 = 0
            if trial % 4 == 3:
                post = np.exp(-rng.uniform(0, 80, size=H))                    # many p_h far below the 1e-12 clamp
            post = post / post.sum()
            row = rng.integers(0, min(C, 11), size=H)
            lit = literal_mp_entropy(row, post, C, gamma)
            grp = grouped_mp_entropy(row, post, C, gamma)
            assert np.isfinite(grp)
            worst = max(worst, abs(lit - grp))
    # the clamp adds at most H * 1e-12 * log2(1e12) ~ H * 4e-11 per class-averaged entropy
    assert worst <= 5e-8, worst


def test_grouped_entropy_ignores_class_ids():
    rng = np.random.default_rng(1)
    H, C = 40, 9
    post = rng.dirichlet(np.ones(H))
    row = rng.integers(0, C, size=H)
    perm = rng.permutation(C)
    assert grouped_mp_entropy(row, post, C, 0.9) == grouped_mp_entropy(perm[row], post, C, 0.9)


def test_grouped_vma_sum_equals_the_pairwise_sum():
    rng = np.random.default_rng(2)
    for H, C in ((8, 3), (30, 10), (64, 100)):
        for _ in range(20):
            pbar = rng.dirichlet(np.ones(C)).astype(np.float32)
            row = rng.integers(0, min(C, 7), size=H)
            l = 1.0 - pbar[row]
            pairwise = sum(abs(float(l[i]) - float(l[j])) for i, j in itertools.combinations(range(H), 2))
            cls, m = np.unique(row, return_counts=True)
            lk = 1.0 - pbar[cls]
            grouped = sum(m[i] * m[j] * abs(float(lk[i]) - float(lk[j]))
                          for i, j in itertools.combinations(range(len(cls)), 2))
            assert abs(pairwise - grouped) <= 1e-9 * max(1.0, pairwise)
            assert abs(float(l.astype(np.float64).sum()) - float((m * lk.astype(np.float64)).sum())) < 1e-9


def draw_model(weights, labeled, u, chunk=4096, ipt=16):
    """k_wsum_blocks + k_wdraw_xchg on one shard: fp64 sums per thread run, per block, then the first item with cum > u * total."""
    n = len(weights)
    items = [i for i in range(n) if not labeled[i]]
    blocks = []
    for lo in range(0, n, chunk):
        runs = [sum(float(weights[i]) for i in range(t, min(n, t + ipt)) if not labeled[i])
                for t in range(lo, min(n, lo + chunk), ipt)]
        blocks.append(sum(runs))
    target = u * sum(blocks)
    base = 0.0
    for b, s in enumerate(blocks):
        if base + s > target:
            cum = base
            for i in range(b * chunk, min(n, (b + 1) * chunk)):
                if labeled[i]:
                    continue
                cum += float(weights[i])
                if cum > target:
                    return items.index(i), i
            break
        base += s
    return len(items) - 1, items[-1]


def test_weighted_draw_model_picks_what_random_choices_picks():
    rng = np.random.default_rng(3)
    for n in (7, 300, 9000):
        for trial in range(20):
            raw = rng.random(n).astype(np.float32) ** 3
            raw[rng.random(n) < 0.1] = 0
            labeled = rng.random(n) < 0.2
            unl = [i for i in range(n) if not labeled[i]]
            tot = np.float32(raw[unl].astype(np.float64).sum())
            w = (raw / tot).astype(np.float32)                # the fp32 normalisation of activetesting.py:44
            state = random.getstate()
            ref = random.choices(unl, weights=[float(w[i]) for i in unl])[0]
            random.setstate(state)
            pos, idx = draw_model(w, labeled, random.random())
            assert idx == ref and unl[pos] == idx, (n, trial)


def test_unlabeled_items_positional_access():
    from coda_b200.baselines import _UnlabeledItems
    rng = random.Random(4)
    ref = list(range(200))
    marked = []
    u = _UnlabeledItems(200, marked.append)
    for _ in range(150):
        x = rng.choice(ref)
        ref.remove(x)
        u.remove(x)
        k = rng.randrange(len(ref))
        assert u[k] == ref[k] and u[-1] == ref[-1] and u.index(ref[k]) == k and len(u) == len(ref)
    assert list(u) == ref and sorted(marked) == sorted(set(range(200)) - set(ref))


def test_shim_serves_the_gpu_classes_without_a_reference():
    code = (
        "import coda.baselines as b, coda_b200.baselines as ours\n"
        "from coda.baselines.modelpicker import TASK_EPS, ModelPicker\n"
        "assert TASK_EPS == {} and ModelPicker is ours.ModelPicker\n"
        "for n in ('IID', 'Uncertainty', 'ActiveTesting', 'VMA', 'ModelPicker'):\n"
        "    assert getattr(b, n) is getattr(ours, n), n\n"
        "from coda_b200.synth import synth\n"
        "from coda.options import LOSS_FNS\n"
        "p, l = synth(4, 50, 3, 1)\n"
        "class DS: pass\n"
        "d = DS(); d.preds, d.labels, d.device = p, l, p.device\n"
        "for make in (lambda: b.IID(d, LOSS_FNS['acc']), lambda: b.ModelPicker(d), lambda: b.IID(None, None)):\n"
        "    try:\n"
        "        make(); raise SystemExit('constructed on the CPU')\n"
        "    except NotImplementedError as e:\n"
        "        assert 'no CPU path' in str(e) and 'CODA_REFERENCE_PATH' in str(e), e\n"
        "print('OK')\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    env.pop("CODA_REFERENCE_PATH", None)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout + r.stderr[-2000:]
