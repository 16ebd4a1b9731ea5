"""The competing selectors of the paper's comparison -- IID, Uncertainty, ActiveTesting, VMA and ModelPicker (reference
coda/baselines/*.py) -- on the sm_90a kernels of ``csrc/baselines.cu``.

Same constructors, methods, attributes and return types as the reference classes, and the same random-number
consumption call for call (Python ``random``, the torch CPU generator, and the CUDA generator where the reference
passes ``device=``), so that a seeded ``main.py --method ...`` run makes the same draws.  Everything with an item axis
runs in the kernels over the products of one slab scan (``hard``, ``disagree``, ``ens``); the per-label bookkeeping
(losses, risk sums, the LURE estimate, the ModelPicker posterior) is H- or M-sized and stays a few torch ops.

One GPU, dense ``(H, N, C)`` slab.  There is no CPU path: a CPU ``dataset.preds`` raises ``NotImplementedError``.
"""
from __future__ import annotations

import bisect
import random

import numpy as np
import torch

from . import _native as nat
from .base import ModelSelector
from .selector import _Unlabeled

_NO_CPU = ("coda_b200.baselines: dataset.preds must be a CUDA tensor on an sm_90a device; there is no CPU path in this "
           "package (set CODA_REFERENCE_PATH to a checkout of justinkay/coda to use the reference implementation)")


def ensemble_entropy(ens, H):
    """Entropy of the ensemble-mean prediction per item (uncertainty.py:6-11) from the ensemble sums ``ens`` [N][C]."""
    mean = ens / float(H)
    return -(mean * torch.log(mean + 1e-8)).sum(-1)


def _ptr(t):
    return t.data_ptr() if t is not None else None


class _UnlabeledItems(_Unlabeled):
    """``d_u_idxs``: the unlabeled items in ascending order, list-like, with O(labels) positional access."""

    def __init__(self, n, on_remove):
        super().__init__(0, n, on_remove)
        self._sorted = []

    def remove(self, idx):
        super().remove(idx)
        bisect.insort(self._sorted, int(idx))

    def __getitem__(self, k):
        n = len(self)
        k = int(k)
        if k < 0:
            k += n
        if not 0 <= k < n:
            raise IndexError("list index out of range")
        for r in self._sorted:                      # ascending: every removed item at or below the answer shifts it
            if r > k:
                break
            k += 1
        return k

    def index(self, idx):
        if idx not in self:
            raise ValueError(f"{idx} is not in list")
        return int(idx) - bisect.bisect_left(self._sorted, int(idx))


class _DeviceState:
    """What the selectors keep on the device: the slab scan, the ``labeled`` mask, the selection scratch and a flags
    word.  Work is enqueued on the device's current stream."""

    def __init__(self, dataset):
        from .datasets import CompactSlab
        from .dist import default_comm
        preds = getattr(dataset, "preds", None)
        if isinstance(preds, CompactSlab):
            raise NotImplementedError("coda_b200.baselines: the compact slab is not supported; use a dense slab")
        if not isinstance(preds, torch.Tensor) or not preds.is_cuda:
            raise NotImplementedError(_NO_CPU)
        if default_comm().world > 1:
            raise NotImplementedError("coda_b200.baselines: one process per GPU (a torch.distributed group of world > 1) "
                                      "is not supported; the baselines run on one GPU")
        self.fmt = nat.slab_format(preds.dtype)      # float32, float16 or bfloat16 (read at its stored width)
        if preds.dim() != 3:
            raise TypeError("coda_b200: preds must be an (H, N, C) tensor (coda/datasets.py:14)")
        H, N, C = (int(s) for s in preds.shape)
        if int(getattr(dataset, "n_global", N)) != N:
            raise NotImplementedError("coda_b200.baselines: an N-range shard of a task is not supported; the baselines "
                                      "need all items on one GPU")
        if not (preds.stride(2) == 1 and preds.stride(1) == C and (H == 1 or preds.stride(0) >= N * C)):
            raise ValueError("coda_b200: preds must be (H, N, C) with contiguous items")
        if H > 1024:
            raise NotImplementedError("coda_b200: H > 1024 models is not supported yet")
        self.lib = nat.load()
        self.preds, self.dev = preds, preds.device
        self.H, self.N, self.C = H, N, C
        self.model_stride = int(preds.stride(0)) if H > 1 else N * C
        with torch.cuda.device(self.dev):
            nat.require_device()
            nb = int(self.lib.coda_b200_select_blocks(N))
            self.labeled = torch.zeros(N, dtype=torch.uint8, device=self.dev)
            self.flags = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self.part_i = torch.empty(2 * nb, dtype=torch.int64, device=self.dev)
            self.part_f = torch.empty(2 * nb, dtype=torch.float64, device=self.dev)
            self.best = torch.empty(2, dtype=torch.int64, device=self.dev)
            self.out = torch.empty(3, dtype=torch.int64, device=self.dev)
            self.total_buf = torch.empty(2, dtype=torch.float64, device=self.dev)

    def _s(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def _call(self, name, *args):
        nat.check(getattr(self.lib, name)(*args), name)

    def scan(self, ens=False):
        """One pass over the slab -> (hard [N][H] u16 bits as int16, disagree [N] u8, ens [N][C] or None)."""
        H, N, C = self.H, self.N, self.C
        with torch.cuda.device(self.dev):
            hard = torch.empty((N, H), dtype=torch.int16, device=self.dev)
            pseudo = torch.empty(N, dtype=torch.int32, device=self.dev)
            disagree = torch.empty(N, dtype=torch.uint8, device=self.dev)
            e = torch.empty((N, C), dtype=torch.float32, device=self.dev) if ens else None
            if self.fmt == nat.SLAB_F32:
                self._call("coda_b200_scan_slab", _ptr(self.preds), self.model_stride, H, N, C, _ptr(hard), _ptr(pseudo),
                           _ptr(disagree), _ptr(e), _ptr(self.flags), self._s())
            else:
                self._call("coda_b200_scan_slab_x", _ptr(self.preds), self.fmt, self.model_stride, H, N, C, _ptr(hard),
                           _ptr(pseudo), _ptr(disagree), _ptr(e), _ptr(self.flags), self._s())
            flags = int(self.flags.item())
        if flags & nat.FLAG_NONFINITE_INPUT:
            raise RuntimeError("[NUMERIC ERROR] preds has bad values (NaN/Inf)")
        if flags & nat.FLAG_RANGE_INPUT:
            raise ValueError("coda_b200: dataset.preds must hold post-softmax scores in [0, 1] (coda/datasets.py:6)")
        return hard, disagree, e

    def static_scores(self, hard, ens, vma):
        with torch.cuda.device(self.dev):
            out = torch.empty(self.N, dtype=torch.float32, device=self.dev)
            self._call("coda_b200_static_scores", _ptr(hard), _ptr(ens), self.H, self.N, self.C,
                       None if vma else _ptr(out), _ptr(out) if vma else None, self._s())
        return out

    def mark(self, idx):
        with torch.cuda.device(self.dev):
            self.labeled[idx] = 1

    def extreme(self, v, want_max):
        """-> (best value over the unlabeled items as a float, number of items exactly equal to it)."""
        with torch.cuda.device(self.dev):
            self._call("coda_b200_select_extreme", _ptr(v), _ptr(self.labeled), self.N, int(want_max),
                       _ptr(self.part_i), _ptr(self.best), self._s())
            bits, cnt = self.best.tolist()
        return float(np.array([bits], dtype=np.int64).astype(np.uint32).view(np.float32)[0]), int(cnt)

    def kth(self, v, k):
        """The k-th unlabeled item (ascending index) equal to the value of the last ``extreme`` call."""
        with torch.cuda.device(self.dev):
            self._call("coda_b200_select_kth", _ptr(v), _ptr(self.labeled), self.N, _ptr(self.part_i), _ptr(self.best),
                       int(k), _ptr(self.out), self._s())
            idx = int(self.out[0].item())
        if idx < 0:
            raise RuntimeError(f"coda_b200: select_kth found no item {k}")
        return idx

    def total(self, w):
        """-> (fp64 sum of w over the unlabeled items, their count)."""
        with torch.cuda.device(self.dev):
            self._call("coda_b200_weighted_total", _ptr(w), _ptr(self.labeled), self.N, _ptr(self.part_f),
                       _ptr(self.total_buf), self._s())
            s, n = self.total_buf.tolist()
        return s, int(n)

    def draw(self, w, u):
        """random.choices over the unlabeled items with weights w / total (after ``total``) -> (item, its weight)."""
        with torch.cuda.device(self.dev):
            self._call("coda_b200_weighted_draw", _ptr(w), _ptr(self.labeled), self.N, _ptr(self.total_buf), float(u),
                       _ptr(self.part_f), _ptr(self.out), self._s())
            _pos, idx, qbits = self.out.tolist()
        return int(idx), float(np.array([qbits], dtype=np.int64).astype(np.uint32).view(np.float32)[0])

    def close(self):
        for k, v in list(self.__dict__.items()):
            if isinstance(v, torch.Tensor):
                setattr(self, k, None)


class _Baseline(ModelSelector):
    def _setup(self, dataset):
        if dataset is None:
            raise NotImplementedError(_NO_CPU)
        self.state = _DeviceState(dataset)
        self.dataset = dataset
        self.device = dataset.preds.device
        self.H, self.N, self.C = self.state.H, self.state.N, self.state.C
        self.d_l_idxs = []
        self.d_l_ys = []
        self.d_u_idxs = _UnlabeledItems(self.N, self.state.mark)

    def _record(self, chosen_idx, true_class):
        self.d_u_idxs.remove(chosen_idx)
        self.d_l_idxs.append(chosen_idx)
        self.d_l_ys.append(true_class)

    def _min_risk_model(self, risk):
        """Lowest risk, a uniformly drawn one of the exact ties (torch.randperm on the CPU generator) -> 0-d tensor."""
        best_risk, best = torch.min(risk, dim=0)
        ties = risk == best_risk
        if ties.sum() > 1:
            idxs = torch.nonzero(ties, as_tuple=True)[0]
            best = idxs[torch.randperm(len(idxs))[0]]
            self.stochastic = True
        return best

    def close(self):
        """Free the device buffers now (a script can then build the next selector on the same card)."""
        if getattr(self, "state", None) is not None:
            self.state.close()
        self.state = None
        self.dataset = None


class IID(_Baseline):
    """Uniform sampling of the unlabeled items; the best model has the lowest mean loss on the labels (iid.py)."""

    def __init__(self, dataset, loss_fn):
        self._setup(dataset)
        self.loss_fn = loss_fn
        self.stochastic = True
        self._risk_sum = torch.zeros(self.H, device=self.device)

    def get_next_item_to_label(self):
        self.stochastic = True
        n = len(self.d_u_idxs)
        idx = self.d_u_idxs[random.choice(range(n))]      # the same draw as random.choice over the list
        return idx, 1.0 / n

    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        # the per-label losses added in label order: the sum iid.py:37-43 recomputes from scratch
        # (a 16-bit slab's scores are widened first: the loss sees the fp32 values the reference loader would produce)
        self._risk_sum += self.loss_fn(self.dataset.preds[:, chosen_idx, :].float(),
                                       torch.tensor([true_class], device=self.device).expand(self.H))

    def get_risk_estimates(self):
        risk = self._risk_sum.clone()
        if self.d_l_idxs:
            risk /= len(self.d_l_idxs)
        return risk

    def get_best_model_prediction(self):
        return self._min_risk_model(self.get_risk_estimates())


class Uncertainty(IID):
    """The unlabeled item of highest ensemble-mean entropy (uncertainty.py); a static score."""

    def __init__(self, dataset, loss_fn):
        super().__init__(dataset, loss_fn)
        _hard, _dis, ens = self.state.scan(ens=True)
        self.score = ensemble_entropy(ens, self.H)
        del _hard, _dis, ens
        self.stochastic = False

    def get_next_item_to_label(self):
        if not len(self.d_u_idxs):
            raise IndexError("max(): Expected reduction dim 0 to have non-zero size.")
        val, cnt = self.state.extreme(self.score, want_max=True)
        k = 0
        if cnt > 1:
            self.stochastic = True
            k = int(torch.randperm(cnt)[0])
        return self.state.kth(self.score, k), val


class ActiveTesting(IID):
    """Kossen et al. (2021): items drawn with probability proportional to the expected loss under the ensemble-mean
    surrogate, summed over the models; risks by the LURE estimator (activetesting.py)."""

    _vma = False

    def __init__(self, dataset, loss_fn):
        super().__init__(dataset, loss_fn)
        hard, _dis, ens = self.state.scan(ens=True)
        self.score = self.state.static_scores(hard, ens, vma=self._vma)
        del hard, _dis, ens
        self.M = 0
        self.losses = []
        self.qs = []
        self.stochastic = True

    def _draw(self):
        total, n = self.state.total(self.score)
        if n == 0:
            raise IndexError("list index out of range")
        if not np.float32(total) > 0:                     # the normalised weights are 0 / 0
            raise ValueError("Total of weights must be finite")
        return self.state.draw(self.score, random.random())

    def get_next_item_to_label(self):
        return self._draw()

    def get_vs(self):
        """LURE weights v_m (Farquhar et al. 2021) of the labels so far, m = 1 .. M."""
        N, M = self.N, self.M
        return [1 + ((N - M) / (N - m)) * (1 / ((N - m + 1) * q) - 1) for m, q in enumerate(self.qs, start=1)]

    def get_lure_risks_and_vars(self):
        losses = torch.stack(self.losses, dim=1).view(self.H, -1)
        weighted = torch.tensor(self.get_vs(), device=self.device).unsqueeze(0) * losses
        return weighted.mean(dim=1), weighted.var(dim=1, unbiased=True) / self.M

    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        self.losses.append(self.loss_fn(self.dataset.preds[:, chosen_idx, :].float(),
                                        torch.tensor([true_class], device=self.device).repeat(self.H), reduction="none"))
        self.qs.append(selection_prob)
        self.M += 1

    def get_risk_estimates(self):
        return self.get_lure_risks_and_vars()[0]

    def get_best_model_prediction(self):
        if self.losses:
            return self._min_risk_model(self.get_risk_estimates())
        return torch.arange(self.H, device=self.device)[random.choice(range(self.H))]


class VMA(ActiveTesting):
    """Matsuura & Hara (2023): items drawn with probability proportional to sum_{h < h'} |loss_h - loss_h'| under the
    ensemble-mean surrogate (vma.py); uniform when every score is 0."""

    _vma = True

    def get_next_item_to_label(self):
        total, n = self.state.total(self.score)
        if np.float32(total) < np.float32(1e-12):
            return self.d_u_idxs[random.choice(range(n))], 1.0 / n
        return self.state.draw(self.score, random.random())


class ModelPicker(_Baseline):
    """Karimi et al. (2021): the unlabeled item of least expected posterior entropy over the models, the best model
    the one with the most correct labels (modelpicker.py)."""

    def __init__(self, dataset, epsilon=0.46):
        self._setup(dataset)
        self.hard, disagree, _ = self.state.scan(ens=False)
        self.disagree = disagree
        self._disagree_host = disagree.cpu().numpy()
        self._n_disagree = int(self._disagree_host.sum())     # unlabeled items some model disagrees on
        self.epsilon = float(epsilon)
        self.gamma = (1.0 - self.epsilon) / self.epsilon
        self.posterior = torch.ones(self.H, device=self.device) / self.H
        self.correct_counts = torch.zeros(self.H, dtype=torch.long, device=self.device)
        self.entropies = torch.empty(self.N, dtype=torch.float32, device=self.device)
        self.stochastic = True

    def get_next_item_to_label(self):
        n = len(self.d_u_idxs)
        if n == 0:
            raise RuntimeError("min(): Expected reduction dim to be specified for input.numel() == 0.")
        st = self.state
        with torch.cuda.device(st.dev):
            # gamma enters modelpicker.py:78 as a float32 factor
            st._call("coda_b200_mp_entropy", _ptr(self.hard), _ptr(self.posterior), self.H, self.N, self.C,
                     float(np.float32(self.gamma)), _ptr(st.labeled), _ptr(self.disagree), int(self._n_disagree > 0),
                     _ptr(self.entropies), st._s())
        _val, cnt = st.extreme(self.entropies, want_max=False)
        k = int(torch.randint(cnt, (1,))[0])                 # drawn every step, one tie or many (modelpicker.py:70)
        return st.kth(self.entropies, k), 1.0 / float(n)

    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        if self._disagree_host[int(chosen_idx)]:
            self._n_disagree -= 1
        preds = self.dataset.preds[:, chosen_idx].argmax(dim=1)
        self.correct_counts += (preds == true_class).long()
        self.posterior = self.update_posterior(self.posterior, preds, true_class, self.gamma)

    def update_posterior(self, posterior, predictions_i, oracle_i, gamma):
        post = posterior * (gamma ** (predictions_i == oracle_i).float())
        return post / post.sum()

    def get_best_model_prediction(self):
        if not self.d_l_idxs:
            return torch.randint(self.H, (1,), device=self.device).item()
        ties = torch.nonzero(self.correct_counts == torch.max(self.correct_counts)).flatten()
        return ties[torch.randint(len(ties), (1,), device=self.device)].item()


__all__ = ["IID", "Uncertainty", "ActiveTesting", "VMA", "ModelPicker", "ensemble_entropy"]
