"""CPU checks of the device mirror of Python's ``random`` (csrc/pyrandom.cuh) behind ``run_steps(tie_rule="reference")``:
a NumPy restatement of its three-phase twist, ``_randbelow`` and both ``random.sample`` branches against the
interpreter's own generator, the state conversion, and the new ABI entries."""
import os
import random
import re

import numpy as np
import pytest

from helpers import ROOT

N, M = 624, 397


def _twist(mt):
    """The twist as pyrandom.cuh runs it: three phases, every word of a phase computed from the words before it."""
    mt = mt.copy()
    for lo, hi in ((0, 227), (227, 454), (454, N)):
        kk = np.arange(lo, hi)
        y = (mt[kk] & np.uint32(0x80000000)) | (mt[(kk + 1) % N] & np.uint32(0x7fffffff))
        new = mt[(kk + M) % N] ^ (y >> np.uint32(1)) ^ np.where(y & np.uint32(1), np.uint32(0x9908b0df), np.uint32(0))
        mt[kk] = new.astype(np.uint32)
    return mt


class Model:
    def __init__(self, state):
        self.mt = np.array(state[1][:N], dtype=np.uint32)
        self.pos = state[1][N]

    def next(self):
        if self.pos >= N:
            self.mt, self.pos = _twist(self.mt), 0
        y = int(self.mt[self.pos])
        self.pos += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9d2c5680
        y ^= (y << 15) & 0xefc60000
        y ^= y >> 18
        return y & 0xffffffff

    def randbelow(self, n):
        k = n.bit_length()
        r = self.next() >> (32 - k)
        while r >= n:
            r = self.next() >> (32 - k)
        return r

    def sample(self, n, m, setsize):
        if n <= setsize:
            pool = list(range(n))
            out = []
            for i in range(m):
                j = self.randbelow(n - i)
                out.append(pool[j])
                pool[j] = pool[n - i - 1]
            return out
        seen, out = set(), []
        for _ in range(m):
            j = self.randbelow(n)
            while j in seen:
                j = self.randbelow(n)
            seen.add(j)
            out.append(j)
        return out

    def state(self, gauss_next):
        return (3, tuple(int(w) for w in self.mt) + (self.pos,), gauss_next)


NS = [1, 2, 3, 4, 5, 64, 65, 2 ** 20, 2 ** 20 + 1, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1]


@pytest.mark.parametrize("seed", [0, 1, 12345])
def test_randbelow_matches_the_interpreter_across_many_twists(seed):
    random.seed(seed)
    model = Model(random.getstate())
    for rep in range(400):                              # ~12 000 words: many 624-word boundaries
        for n in NS:
            assert model.randbelow(n) == random._inst._randbelow(n), (rep, n)
            if n > 1:
                want = random.choice(range(n))
                assert model.randbelow(n) == want
    assert model.state(random.getstate()[2]) == random.getstate()


def _setsize_cases():
    from coda_b200.selector import sample_setsize
    cases = []
    for m in (1, 5, 6, 7, 50, 333):
        s = sample_setsize(m)
        cases += [(s, m), (s + 1, m), (max(m, s - 1), m)]       # either side of the pool / set switch
    return cases


@pytest.mark.parametrize("n,m", _setsize_cases() + [(10, 10), (1, 1), (2 ** 31 - 1, 40)])
def test_sample_branches_match_the_interpreter(n, m):
    from coda_b200.selector import sample_setsize
    random.seed(n * 7 + m)
    for _ in range(3):                                  # a couple of steps: the state carries over
        model = Model(random.getstate())
        got = model.sample(n, m, sample_setsize(m))
        assert got == random.sample(range(n), m)
        assert model.state(random.getstate()[2]) == random.getstate()


def test_setsize_is_the_interpreters():
    """sample_setsize(m) is the switch of Lib/random.py: a population of setsize items draws from the pool (n - i per
    draw), one more item from the set (n every draw); the first draw's bound tells the two apart."""
    from coda_b200.selector import sample_setsize
    seen = []
    orig = random.Random._randbelow

    def spy(self, n):
        seen.append(n)
        return orig(self, n)
    for m in (1, 6, 30, 400):
        s = sample_setsize(m)
        random.Random._randbelow = spy
        try:
            seen.clear()
            random.sample(range(s), m)
            pool_bounds = list(seen)
            seen.clear()
            random.sample(range(s + 1), m)
            set_bounds = list(seen)
        finally:
            random.Random._randbelow = orig
        assert pool_bounds == [s - i for i in range(m)]
        assert len(set_bounds) >= m and set(set_bounds) == {s + 1}


def test_state_conversion_round_trips():
    from coda_b200.selector import rng_state, rng_words
    for seed in (0, 99):
        random.seed(seed)
        for _ in range(seed):
            random.random()
        st = random.getstate()
        w = rng_words(st)
        assert w.dtype.is_floating_point is False and w.numel() == 625 and int(w[624]) == st[1][624]
        assert rng_state(w, st[2]) == st
    random.seed(5)
    random.gauss(0, 1)                                  # gauss_next is set: it is carried, not taken from the words
    st = random.getstate()
    assert st[2] is not None and rng_state(rng_words(st), st[2]) == st


def test_new_abi_entries_and_their_argument_counts():
    from coda_b200 import _native as nat
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    want = {"coda_b200_step_select_defer": 4, "coda_b200_step_label_if": 4, "coda_b200_tie_band": 8,
            "coda_b200_tie_draw": 9, "coda_b200_pf_sample": 10, "coda_b200_prefilter_commit_defer": 10,
            "coda_b200_pf_band": 14, "coda_b200_pf_tie_max_m": 1, "coda_b200_pf_tie_draw": 9,
            "coda_b200_pyrandom_run": 7}
    for name, n in want.items():
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
        assert m and m.group(1).count(",") + 1 == n == len(nat.SIGNATURES[name][1]), name
    lib = nat.load()
    assert nat.VERSION == 203 and lib.coda_b200_version() == 203
    # the record slot at H = 1: 64 + 2 * 16 bytes, one bit per sample position
    assert lib.coda_b200_pf_tie_max_m(1) == 768 and lib.coda_b200_pf_tie_max_m(256) == 8 * (64 + 2 * 512)


def test_run_steps_rejects_an_unknown_tie_rule():
    from coda_b200.selector import CODA
    sel = CODA.__new__(CODA)
    with pytest.raises(ValueError, match="tie_rule"):
        sel.run_steps(1, None, tie_rule="random")
