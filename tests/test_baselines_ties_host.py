"""CPU checks behind the competing selectors' ``run_steps(..., tie_rule="reference")``: a model of how torch's CPU
generator is consumed by ``randperm`` and ``randint`` (the draws csrc/bl_ref.cu mirrors), against torch itself across
the size thresholds; the state-byte conversion; the CUDA generator's Philox word; the ABI entries; the refusals."""
import os
import re

import numpy as np
import pytest
import torch

from helpers import ROOT
from test_baselines_loop_host import philox4x32_10
from test_coda_loop_ties_host import _twist

N = 624
M32 = 0xFFFFFFFF


class TorchCpuModel:
    """torch's CPU generator from ``torch.get_rng_state()`` bytes: MT19937 with the position pos = 625 - left."""

    def __init__(self, state):
        b = state.numpy().tobytes()
        self.mt = np.frombuffer(b[24:24 + 8 * N], "<u8").astype(np.uint32)
        self.pos = 625 - int(np.frombuffer(b, "<i4", 1, 8)[0])

    def next(self):
        if self.pos >= N:
            self.mt, self.pos = _twist(self.mt), 0
        y = int(self.mt[self.pos])
        self.pos += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9d2c5680
        y ^= (y << 15) & 0xefc60000
        y ^= y >> 18
        return y & M32

    def skip(self, n):
        """n words drawn and dropped, as tc_skip: a twist per 624."""
        while n > 0:
            if self.pos >= N:
                self.mt, self.pos = _twist(self.mt), 0
            a = min(n, N - self.pos)
            self.pos += a
            n -= a

    def randperm(self, n):
        """The whole permutation: Fisher-Yates, z = random() % (n - i) for i < n - 1."""
        r = list(range(n))
        for i in range(n - 1):
            z = self.next() % (n - i)
            r[i], r[i + z] = r[i + z], r[i]
        return r

    def randperm0(self, n):
        """randperm(n)[0] as the device draws it: one word mod n, n - 2 words dropped."""
        if n < 2:
            return 0
        r = self.next() % n
        self.skip(n - 2)
        return r

    def randint(self, n):
        if n >= 1 << 28:
            hi = self.next()
            return ((hi << 32) | self.next()) % n
        return self.next() % n

    def same_as(self, state):
        other = TorchCpuModel(state)
        return other.pos == self.pos and np.array_equal(other.mt, self.mt)


def cuda_randint(seed, offset, n):
    """torch.randint(n, (1,), device="cuda") from {seed, offset} (n < 2^28): curand4 of curand_init(seed, 0, offset) is
    Philox4x32-10 at counter offset / 4, key seed; x % n.  The offset then advances by 4."""
    seed &= (1 << 64) - 1
    c = offset // 4
    return philox4x32_10((c & M32, c >> 32, 0, 0), (seed & M32, seed >> 32))[0] % n


def test_state_layout_after_manual_seed():
    torch.manual_seed(0)
    st = torch.get_rng_state()
    assert st.numel() == 5056
    b = st.numpy().tobytes()
    seed, left, seeded, nxt = (int(np.frombuffer(b, t, 1, o)[0]) for t, o in (("<u8", 0), ("<i4", 8), ("<i4", 12),
                                                                                ("<u8", 16)))
    assert (seed, left, seeded, nxt) == (0, 1, 1, 0)
    assert TorchCpuModel(st).pos == N                       # the next word twists first
    assert not (np.frombuffer(b[24:24 + 8 * N], "<u8") >> np.uint64(32)).any()     # words in the low 32 bits


@pytest.mark.parametrize("seed", [0, 7])
def test_randperm_first_element_and_consumption(seed):
    torch.manual_seed(seed)
    model = TorchCpuModel(torch.get_rng_state())
    for n in [2, 3, 5, 64, 623, 624, 625, 1000, 1247, 70_000, 1 << 20, (1 << 20) + 1]:
        assert int(torch.randperm(n)[0]) == model.randperm0(n), n
        assert model.same_as(torch.get_rng_state()), n
    for n in (0, 1):                                        # nothing drawn
        torch.randperm(n)
        assert model.same_as(torch.get_rng_state()), n


def test_randperm_whole_permutation_up_to_300():
    torch.manual_seed(3)
    model = TorchCpuModel(torch.get_rng_state())
    for n in range(1, 301):
        assert torch.randperm(n).tolist() == model.randperm(n), n
    assert model.same_as(torch.get_rng_state())


def test_randint_across_the_64_bit_switch():
    torch.manual_seed(11)
    model = TorchCpuModel(torch.get_rng_state())
    for rep in range(3):
        for n in [1, 2, 3, 1000, (1 << 28) - 1, 1 << 28, (1 << 28) + 1, M32, 1 << 32, (1 << 40) + 3, (1 << 62) + 5]:
            assert int(torch.randint(n, (1,))[0]) == model.randint(n), (rep, n)
            assert model.same_as(torch.get_rng_state()), (rep, n)


def test_randperm_switch_constant():
    """randperm_cpu takes 32-bit words while n < UINT32_MAX / 20; the C header and the binding agree."""
    from coda_b200 import _native as nat
    hdr = open(os.path.join(ROOT, "include", "coda_b200.h")).read()
    m = re.search(r"#define CODA_B200_RANDPERM32_MAX (\d+)LL", hdr)
    assert int(m.group(1)) == nat.RANDPERM32_MAX == (2 ** 32 - 1) // 20


def test_state_bytes_round_trip():
    from coda_b200.baselines import torch_rng_state, torch_rng_words
    torch.manual_seed(5)
    torch.randn(3)                                          # the normal sampler's cache is set: carried as is
    for draws in (0, 1, 623, 624, 625, 2000):
        st = torch.get_rng_state()
        words = torch_rng_words(st)
        assert words.dtype == torch.int32 and words.numel() == 625
        back = torch_rng_state(words, st)
        assert torch.equal(back, st), draws
        # the replica advanced by the model, written back, equals torch advanced by itself, byte for byte
        model = TorchCpuModel(st)
        model.skip(draws)
        w = np.empty(625, np.uint32)
        w[:N], w[N] = model.mt, model.pos
        got = torch_rng_state(torch.from_numpy(w.view(np.int32)), st)
        torch.randperm(draws + 1)                           # draws words
        assert torch.equal(got, torch.get_rng_state()), draws
        torch.set_rng_state(got)
        assert torch.equal(torch.get_rng_state(), got)


def test_right_after_manual_seed_the_position_maps_back():
    """left = 1, next = 0 (as manual_seed leaves it) reads as pos 624; words written back after a draw are torch's."""
    from coda_b200.baselines import torch_rng_state, torch_rng_words
    torch.manual_seed(9)
    st = torch.get_rng_state()
    w = torch_rng_words(st)
    assert int(w[624]) == N
    model = TorchCpuModel(st)
    r = model.randint(10)
    assert int(torch.randint(10, (1,))[0]) == r
    ww = np.empty(625, np.uint32)
    ww[:N], ww[N] = model.mt, model.pos
    assert torch.equal(torch_rng_state(torch.from_numpy(ww.view(np.int32)), st), torch.get_rng_state())


def test_cuda_state_conversion_and_word_model():
    from coda_b200.baselines import cuda_rng_state, cuda_rng_words
    st = torch.from_numpy(np.array([(1 << 64) - 3, 4 * 12345], "<u8").view(np.uint8).copy())
    w = cuda_rng_words(st)
    assert w.dtype == torch.int64 and w.tolist() == [-3, 4 * 12345]
    assert torch.equal(cuda_rng_state(w), st)
    # curand4 at offset 0 of key 0 is Random123's known answer's first word
    assert cuda_randint(0, 0, 1 << 27) == 0x6627E8D5 % (1 << 27)
    assert cuda_randint(-1, 8, 7) == philox4x32_10((2, 0, 0, 0), (M32, M32))[0] % 7


def test_new_abi_entries_and_their_argument_counts():
    from coda_b200 import _native as nat
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    want = {"coda_b200_bl_draw_ref": 3, "coda_b200_bl_best_ref": 4, "coda_b200_torch_rng_run": 6}
    for name, n in want.items():
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
        assert m and m.group(1).count(",") + 1 == n == len(nat.SIGNATURES[name][1]), name
    lib = nat.load()
    for name in want:
        assert hasattr(lib, name)
    assert nat.VERSION == 203 and lib.coda_b200_version() == 203
    assert len(nat.BlLoopStruct._fields_) == 27             # coda_bl_loop_t is unchanged


@pytest.mark.parametrize("cls", ["IID", "Uncertainty", "ActiveTesting", "VMA", "ModelPicker"])
def test_run_steps_refuses_bad_tie_rule_arguments(cls):
    import coda_b200
    sel = getattr(coda_b200, cls).__new__(getattr(coda_b200, cls))
    with pytest.raises(ValueError, match="tie_rule"):
        sel.run_steps(1, None, tie_rule="first")
    with pytest.raises(ValueError, match="seed"):
        sel.run_steps(1, None, seed=3, tie_rule="reference")


def test_uncertainty_refuses_randperm_sizes_past_the_32_bit_branch():
    from coda_b200 import Uncertainty, _native as nat
    sel = Uncertainty.__new__(Uncertainty)
    sel.N = nat.RANDPERM32_MAX
    with pytest.raises(NotImplementedError, match="randperm"):
        sel._reference_refusals()
    sel.N = nat.RANDPERM32_MAX - 1
    sel._reference_refusals()
