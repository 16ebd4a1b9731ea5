"""CPU tests of the competing selectors' host-free loop: the Philox tie stream, the LURE running sums, the
pre-draw / rewind of Python ``random`` and the C ABI of the loop entry points."""
import os
import random
import re

import numpy as np
import pytest

from helpers import ROOT

M32 = 0xFFFFFFFF


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al. 2011, Random123), as curand_Philox4x32_10: 4 x u32 counter, 2 x u32 key."""
    c0, c1, c2, c3 = (int(v) & M32 for v in ctr)
    k0, k1 = (int(v) & M32 for v in key)
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & M32, p1 & M32, ((p0 >> 32) ^ c3 ^ k1) & M32, p0 & M32
    return c0, c1, c2, c3


def tie_pick(seed, label_count, purpose, cnt):
    """The tie (ascending index order) the device draws among ``cnt`` exact ties (include/coda_b200.h)."""
    seed &= (1 << 64) - 1
    r = philox4x32_10((label_count, purpose, 0, 0), (seed & M32, seed >> 32))
    return (r[0] * cnt) >> 32


def test_philox_model_reproduces_the_random123_known_answers():
    assert philox4x32_10((0, 0, 0, 0), (0, 0)) == (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)
    assert philox4x32_10((M32,) * 4, (M32, M32)) == (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)
    assert philox4x32_10((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0)) == \
        (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)


def test_tie_rule_is_uniform_and_in_range():
    for cnt in (2, 3, 7, 1000, (1 << 40) - 3):
        picks = [tie_pick(12345, c, 0, cnt) for c in range(400)]
        assert all(0 <= p < cnt for p in picks)
    counts = np.bincount([tie_pick(99, c, 1, 4) for c in range(4000)], minlength=4)
    assert counts.min() > 900                                 # ~1000 each
    r = philox4x32_10((5, 1, 0, 0), (7, 0))
    assert tie_pick(7, 5, 1, 10) == (r[0] * 10) >> 32
    assert tie_pick(-1, 0, 0, 3) == tie_pick((1 << 64) - 1, 0, 0, 3)


def _vs(N, qs):
    M = len(qs)
    return [1 + ((N - M) / (N - m)) * (1 / ((N - m + 1) * q) - 1) for m, q in enumerate(qs, start=1)]


def test_lure_identity_equals_the_weighted_sum():
    """sum_m v_m L_m = S1 + (N - M) S2 with S2 = sum_m L_m a_m / (N - m), a_m = 1 / ((N - m + 1) q_m) - 1: the running
    sums bl_step keeps give the get_vs()-weighted sums of activetesting.py in fp64."""
    rng = np.random.default_rng(3)
    for N, M, H in ((500, 40, 12), (10_000, 300, 64), (50, 49, 5)):
        qs = list(rng.uniform(1e-4, 0.05, M))
        L = rng.integers(0, 2, (M, H)).astype(np.float64)
        direct = (np.array(_vs(N, qs))[:, None] * L).sum(0)
        s1, s2 = np.zeros(H), np.zeros(H)
        for m, q in enumerate(qs, start=1):
            t = (1.0 / ((N - m + 1.0) * q) - 1.0) / (N - m)
            s1 = s1 + L[m - 1]
            s2 = s2 + np.where(L[m - 1] != 0, t, 0.0)
        np.testing.assert_allclose(s1 + (N - M) * s2, direct, rtol=1e-12, atol=0)


@pytest.mark.parametrize("kind", ["choice", "random"])
def test_rewind_leaves_the_state_of_j_api_draws(kind):
    from coda_b200.baselines import predraw, rewind
    k, n0 = 25, 700
    random.seed(11)
    state0 = random.getstate()
    pre = predraw(kind, k, n0)
    random.setstate(state0)
    for j in range(k + 1):
        random.setstate(state0)
        api = []
        for s in range(j):                                     # the API path's own calls
            api.append(float(random.choice(range(n0 - s))) if kind == "choice" else random.random())
        want = random.getstate()
        assert api == pre[:j]
        random.seed(999)                                      # anything in between
        rewind(state0, kind, j, n0)
        assert random.getstate() == want, j
    assert predraw(None, k, n0) == []


def test_loop_entry_points_are_declared_and_bound():
    from coda_b200 import _native as nat
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    declared = set(re.findall(r"\b(coda_b200_[a-z0-9_]+)\s*\(", hdr))
    assert declared == set(nat.SIGNATURES)
    for name in ("coda_b200_select_kth_xchg_dev", "coda_b200_weighted_draw_xchg_dev", "coda_b200_mp_entropy_dev",
                 "coda_b200_bl_draw", "coda_b200_bl_step"):
        assert name in nat.SIGNATURES
    lib = nat.load()
    for name in nat.SIGNATURES:
        assert hasattr(lib, name)
    fields = re.search(r"typedef struct coda_bl_loop \{(.*?)\} coda_bl_loop_t;", hdr, flags=re.S).group(1)
    names = []
    for decl in fields.split(";"):
        decl = decl.strip()
        if decl:
            rest = decl[len("const "):] if decl.startswith("const ") else decl
            names += [n.strip(" *") for n in rest.split(None, 1)[1].split(",")]
    assert names == [f[0] for f in nat.BlLoopStruct._fields_]
