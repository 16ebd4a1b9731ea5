"""The competing selectors of the paper's comparison -- IID, Uncertainty, ActiveTesting, VMA and ModelPicker (reference
coda/baselines/*.py) -- on the sm_90a kernels of ``csrc/baselines.cu``.

Same constructors, methods, attributes and return types as the reference classes, and the same random-number
consumption call for call (Python ``random``, the torch CPU generator, and the CUDA generator where the reference
passes ``device=``), so that a seeded ``main.py --method ...`` run makes the same draws.  Everything with an item axis
runs in the kernels over the products of one slab scan (``hard``, ``disagree``, ``ens``); the per-label bookkeeping
(losses, risk sums, the LURE estimate, the ModelPicker posterior) is H- or M-sized and stays a few torch ops.

Dense ``(H, N, C)`` slab (fp32, fp16 or bf16) or ``CompactSlab``.  There is no CPU path: a CPU ``dataset.preds`` raises
``NotImplementedError``.

N-axis shards, as for ``CODA`` (``dist.py``): keyword-only ``gpus=`` / ``shards=`` (or ``CODA_B200_GPUS``) split the
task over GPUs driven by this process (shards may share a GPU, each on its own stream); under ``torch.distributed``
with world > 1 the dataset is this rank's N-range and every rank makes the same calls.  One shard unless asked: there
is no size-based rule.  Each selection call ends in one exchange kernel per shard (``*_xchg`` entry points) that
leaves the same global answer on every shard; ``add_label`` ships the owner's hard row or losses the same way.  The
host bookkeeping (``d_u_idxs``, risks, the posterior, RNG draws) is global and replicated.
"""
from __future__ import annotations

import bisect
import contextlib
import os
import random

import numpy as np
import torch

from . import _native as nat
from .base import ModelSelector
from .dist import InProcessGroup, ProcessGroup, SoloGroup, default_comm, split_slab
from .selector import _Unlabeled

_NO_CPU = ("coda_b200.baselines: dataset.preds must be a CUDA tensor on an sm_90a device; there is no CPU path in this "
           "package (set CODA_REFERENCE_PATH to a checkout of justinkay/coda to use the reference implementation)")


def ensemble_entropy(ens, H):
    """Entropy of the ensemble-mean prediction per item (uncertainty.py:6-11) from the ensemble sums ``ens`` [N][C]."""
    mean = ens / float(H)
    return -(mean * torch.log(mean + 1e-8)).sum(-1)


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _f32(bits):
    return float(np.array([bits], dtype=np.int64).astype(np.uint32).view(np.float32)[0])


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
    """One shard of a selector on the device: the slab scan, the ``labeled`` mask, the selection scratch and a flags
    word.  Work is enqueued on the shard's own stream when it has one, else on the device's current stream.  With
    peers, ``xchg`` / ``_mailbox`` are set by the group (``dist.InProcessGroup`` / ``ProcessGroup``)."""

    rep_words = 8          # the exchanges use the mailbox's record slot; the report slot is kept at its minimum

    def __init__(self, preds, n_offset=0, world=1, own_stream=False):
        from .datasets import CompactSlab
        self.compact = preds if isinstance(preds, CompactSlab) else None
        if not ((isinstance(preds, torch.Tensor) or self.compact is not None) and preds.is_cuda):
            raise NotImplementedError(_NO_CPU)
        H, N, C = (int(s) for s in preds.shape)
        if self.compact is not None:
            self.fmt = None
            self.model_stride = int(preds.ids.stride(0)) if H > 1 else N * preds.K
        else:
            self.fmt = nat.slab_format(preds.dtype)  # float32, float16 or bfloat16 (read at its stored width)
            if preds.dim() != 3:
                raise TypeError("coda_b200: preds must be an (H, N, C) tensor (coda/datasets.py:14)")
            if not (preds.stride(2) == 1 and preds.stride(1) == C and (H == 1 or preds.stride(0) >= N * C)):
                raise ValueError("coda_b200: preds must be (H, N, C) with contiguous items")
            self.model_stride = int(preds.stride(0)) if H > 1 else N * C
        if H > 1024:
            raise NotImplementedError("coda_b200: H > 1024 models is not supported yet")
        self.lib = nat.load()
        self.preds, self.dev = preds, preds.device
        self.H, self.N, self.C = H, N, C
        self.n_offset, self.world = int(n_offset), int(world)
        self.xchg, self._mailbox = None, None
        self.stream = torch.cuda.Stream(device=self.dev) if own_stream else None
        with self._on():
            nat.require_device()
            nb = int(self.lib.coda_b200_select_blocks(N))
            self.labeled = torch.zeros(N, dtype=torch.uint8, device=self.dev)
            self.flags = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self.part_i = torch.empty(2 * nb, dtype=torch.int64, device=self.dev)
            self.part_f = torch.empty(2 * nb, dtype=torch.float64, device=self.dev)
            self.best = torch.empty(4, dtype=torch.int64, device=self.dev)
            self.out = torch.empty(3, dtype=torch.int64, device=self.dev)
            self.total_buf = torch.empty(2, dtype=torch.float64, device=self.dev)

    @contextlib.contextmanager
    def _on(self):
        with torch.cuda.device(self.dev):
            if self.stream is not None:
                with torch.cuda.stream(self.stream):
                    yield
            else:
                yield

    def _s(self):
        return torch.cuda.current_stream(self.dev).cuda_stream

    def _x(self):
        return self.xchg if self.world > 1 else None

    def _call(self, name, *args):
        nat.check(getattr(self.lib, name)(*args), name)

    def enter(self):
        """The shard's stream waits for what the caller's stream has enqueued (inputs the bookkeeping produced)."""
        if self.stream is not None:
            self.stream.wait_stream(torch.cuda.current_stream(self.dev))

    def leave(self):
        """The caller's stream waits for the shard's work (outputs the bookkeeping reads)."""
        if self.stream is not None:
            torch.cuda.current_stream(self.dev).wait_stream(self.stream)

    def scan(self, ens=False):
        """One pass over the slab -> (hard [N][H] u16 bits as int16, disagree [N] u8, ens [N][C] or None)."""
        H, N, C = self.H, self.N, self.C
        with self._on():
            hard = torch.empty((N, H), dtype=torch.int16, device=self.dev)
            pseudo = torch.empty(N, dtype=torch.int32, device=self.dev)
            disagree = torch.empty(N, dtype=torch.uint8, device=self.dev)
            e = torch.empty((N, C), dtype=torch.float32, device=self.dev) if ens else None
            if self.compact is not None:
                cs = self.compact
                self._call("coda_b200_scan_compact", _ptr(cs.ids), _ptr(cs.probs), self.model_stride, H, N, C, cs.K,
                           _ptr(hard), _ptr(pseudo), _ptr(disagree), _ptr(e), _ptr(self.flags), self._s())
            elif self.fmt == nat.SLAB_F32:
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

    def column(self, loc):
        """The (H, C) fp32 scores of local item ``loc`` (a 16-bit slab widened, a compact slab densified)."""
        if self.compact is not None:
            return self.compact.item_column(loc)
        return self.preds[:, loc, :].float()

    def static_scores(self, hard, ens, vma):
        with self._on():
            out = torch.empty(self.N, dtype=torch.float32, device=self.dev)
            self._call("coda_b200_static_scores", _ptr(hard), _ptr(ens), self.H, self.N, self.C,
                       None if vma else _ptr(out), _ptr(out) if vma else None, self._s())
        return out

    def mark(self, idx):
        """Item ``idx`` (global) is labeled: set it in the mask if this shard holds it."""
        loc = int(idx) - self.n_offset
        if 0 <= loc < self.N:
            with self._on():
                self.labeled[loc] = 1

    # -- the selection calls: enqueue only (every shard is enqueued before the host waits on any), then ``read`` -------
    def extreme(self, v, want_max):
        with self._on():
            self._call("coda_b200_select_extreme_xchg", _ptr(v), _ptr(self.labeled), self.N, int(want_max),
                       _ptr(self.part_i), _ptr(self.best), self._x(), _ptr(self.flags), self._s())

    def kth(self, v, k):
        with self._on():
            self._call("coda_b200_select_kth_xchg", _ptr(v), _ptr(self.labeled), self.N, _ptr(self.part_i),
                       _ptr(self.best), int(k), self.n_offset, _ptr(self.out), self._x(), _ptr(self.flags), self._s())

    def total(self, w):
        with self._on():
            self._call("coda_b200_weighted_total_xchg", _ptr(w), _ptr(self.labeled), self.N, _ptr(self.part_f),
                       _ptr(self.total_buf), self._x(), _ptr(self.flags), self._s())

    def draw(self, w, u):
        with self._on():
            self._call("coda_b200_weighted_draw_xchg", _ptr(w), _ptr(self.labeled), self.N, _ptr(self.total_buf),
                       float(u), self.n_offset, _ptr(self.part_f), _ptr(self.out), self._x(), _ptr(self.flags), self._s())

    def share(self, src, own, dst):
        """The owner shard's ``src`` (own = True on exactly one shard) -> ``dst`` on every shard."""
        with self._on():
            self._call("coda_b200_owner_share", _ptr(src) if own else None, dst.numel() * dst.element_size(),
                       int(own), _ptr(dst), self._x(), _ptr(self.flags), self._s())

    def read(self, t):
        """Host copy of ``t`` (a result of the calls above) as a list."""
        with self._on():
            return t.tolist()

    def timed_out(self):
        """True once an exchange of this shard gave up on a peer (the flag is sticky)."""
        with self._on():
            return bool(int(self.flags.item()) & nat.FLAG_XCHG_TIMEOUT)

    def close(self):
        if self._mailbox is not None:
            self._mailbox.close()
            self._mailbox = None
        self.xchg = None
        self.preds = self.compact = None
        for k, v in list(self.__dict__.items()):
            if isinstance(v, torch.Tensor):
                setattr(self, k, None)


def _check_rank_ranges(preds, n_offset, N, n_global, comm):
    """One process per GPU: the ranks' N-ranges must tile [0, n_global) in rank order (the merges take rank order for
    item order); a rank holding the whole task, an overlap or a gap is an error, not a different run."""
    meta = comm.allgather(torch.tensor([n_offset, N, n_global], dtype=torch.int64, device=preds.device)).cpu().tolist()
    lo = 0
    for r, (off, n, ng) in enumerate(meta):
        if off != lo or ng != n_global:
            raise ValueError(f"coda_b200.baselines: under torch.distributed every rank holds its own N-range of the task "
                             f"in rank order; rank {r} has items [{off}, {off + n}) of {ng}, expected to start at {lo} "
                             f"of {n_global} (e.g. SyntheticDataset(..., rank=rank, world=world), ShardedFileDataset)")
        lo += n
    if lo != n_global:
        raise ValueError(f"coda_b200.baselines: the ranks' N-ranges cover {lo} of the task's {n_global} items")


def _layout(dataset, gpus, shards, comm):
    """-> (group, [(shard slab, n_offset)] of this process)."""
    from .datasets import CompactSlab
    preds = getattr(dataset, "preds", None)
    if not ((isinstance(preds, torch.Tensor) or isinstance(preds, CompactSlab)) and preds.is_cuda):
        raise NotImplementedError(_NO_CPU)
    n_offset = int(getattr(dataset, "n_offset", 0))
    N = int(preds.shape[1])
    n_global = int(getattr(dataset, "n_global", N))
    if comm.world > 1:                                     # one process per GPU: this is one shard of the task
        if gpus or shards:
            raise ValueError("coda_b200.baselines: gpus= / shards= split a task inside one process; under "
                             "torch.distributed with world > 1 every rank is one shard (pass this rank's N-range)")
        _check_rank_ranges(preds, n_offset, N, n_global, comm)
        return ProcessGroup(comm), [(preds, n_offset)]
    if n_global != N:
        raise NotImplementedError("coda_b200.baselines: an N-range shard of a task needs its peers: run one process "
                                  "per shard under torch.distributed, or pass the whole task with gpus= / shards=")
    env = os.environ.get("CODA_B200_GPUS")
    nshards = int(shards) if shards else (int(gpus) if gpus else (max(1, int(env)) if env else 1))
    ngpus = int(gpus) if gpus else min(nshards, max(1, torch.cuda.device_count()))
    nshards = max(1, min(nshards, N))
    if nshards == 1:
        return SoloGroup(), [(preds, n_offset)]
    return InProcessGroup(nshards), split_slab(preds, nshards, ngpus)


class _Baseline(ModelSelector):
    def _setup(self, dataset, gpus=None, shards=None, comm=None):
        if dataset is None:
            raise NotImplementedError(_NO_CPU)
        self.group, layout = _layout(dataset, gpus, shards, comm or default_comm())
        own = len(layout) > 1
        self.states = [_DeviceState(p, off, self.group.world, own) for p, off in layout]
        self.state = self.states[0]
        self.group.attach(self.states)
        self._xs = self.group.world > 1                    # selections go through the exchange kernels
        self.dataset = dataset
        self.device = dataset.preds.device
        self.H, self.C = self.state.H, self.state.C
        self.N = int(getattr(dataset, "n_global", dataset.preds.shape[1]))     # callers see the whole task
        self.d_l_idxs = []
        self.d_l_ys = []
        self.d_u_idxs = _UnlabeledItems(self.N, self._mark)

    def _mark(self, idx):
        for st in self.states:
            st.mark(idx)

    def _cat(self, name):
        """Per-item vector ``name`` of the shards of this process, in item order, on the dataset's device."""
        if len(self.states) == 1:
            return getattr(self.state, name)
        for st in self.states:
            st.leave()
        return torch.cat([getattr(st, name).to(self.device) for st in self.states], 0)

    # per-item vectors over this process's items (one process per GPU: this rank's N-range)
    score = property(lambda self: self._cat("score"))
    hard = property(lambda self: self._cat("hard"))
    disagree = property(lambda self: self._cat("disagree"))
    entropies = property(lambda self: self._cat("ent"))

    def _check_exchanges(self):
        """Raise if an exchange of any shard of this process timed out (its outputs are then not valid).  One shard
        has no peer to wait for, so there is no flag to read."""
        if self._xs and any(st.timed_out() for st in self.states):
            raise RuntimeError("coda_b200.baselines: a peer shard did not reach an exchange within 2 s")

    def _read(self, t):
        """Host copy of a global result held by shard 0 (every shard holds the same), after every shard's exchange
        is checked."""
        vals = self.state.read(t)
        self._check_exchanges()
        return vals

    def _select_extreme(self, name, want_max, draw_k):
        """Arg-extreme of per-item vector ``name`` with the k-th tie drawn by ``draw_k(count)`` on the host -> (global
        item, extreme value)."""
        for st in self.states:
            st.enter()
            st.extreme(getattr(st, name), want_max)
        bits, cnt = self._read(self.state.best[:2])
        k = draw_k(int(cnt))
        for st in self.states:
            st.kth(getattr(st, name), k)
        idx = int(self._read(self.state.out[:1])[0])
        if idx < 0:
            raise RuntimeError(f"coda_b200: select_kth found no item {k}")
        return idx, _f32(bits)

    def _total(self):
        for st in self.states:
            st.enter()
            st.total(st.score)
        s, n = self._read(self.state.total_buf)
        return s, int(n)

    def _weighted_draw(self, u):
        for st in self.states:
            st.draw(st.score, u)
        _pos, idx, qbits = self._read(self.state.out)
        return int(idx), _f32(qbits)

    def _share(self, idx, payload, dst_name):
        """add_label on shards: the shard holding item ``idx`` sends ``payload(state, local index)`` (an H-sized tensor on
        its device, cast to the buffer's dtype) to every shard's buffer ``dst_name`` -> that buffer of shard 0, ordered on
        the caller's stream.  The payload is computed before any shard enqueues its exchange: a kernel launched for the first time needs its
        module loaded (CUDA lazy loading), which can wait for a peer's exchange kernel that is already spinning."""
        srcs = []
        for st in self.states:
            st.enter()
            loc = int(idx) - st.n_offset
            src = None
            if 0 <= loc < st.N:
                dst = getattr(st, dst_name)
                with st._on():
                    src = payload(st, loc)
                if src.numel() != dst.numel():
                    raise ValueError(f"coda_b200.baselines: add_label needs {dst.numel()} values per item, got a "
                                     f"tensor of shape {tuple(src.shape)}")
                with st._on():
                    src = src.reshape(-1).to(dst.dtype).contiguous()
            srcs.append(src)
        for st, src in zip(self.states, srcs):             # the exchanges back to back, nothing launched in between
            st.share(src, src is not None, getattr(st, dst_name))
        self.state.leave()
        self._check_exchanges()
        return getattr(self.state, dst_name)

    def _label_losses(self, idx, true_class):
        """The H per-model losses of item ``idx`` (``_loss`` on its (H, C) scores) on the dataset's device.  On shards
        they travel as fp32 (the dtype ``_risk_sum`` and the LURE sums keep); a loss of another dtype is rounded to it."""
        if not self._xs:
            return self._loss(self.state.column(int(idx)), true_class, self.device)
        for st in self.states:
            if getattr(st, "losses_in", None) is None:
                with st._on():
                    st.losses_in = torch.empty(self.H, dtype=torch.float32, device=st.dev)
        got = self._share(idx, lambda st, loc: self._loss(st.column(loc), true_class, st.dev).reshape(-1),
                          "losses_in")
        return got.clone()

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
        """Free the device buffers and mailboxes of every shard now (a script can then build the next selector on the
        same card)."""
        states = getattr(self, "states", None) or ([self.state] if getattr(self, "state", None) is not None else [])
        for st in states:
            if st.stream is not None:
                st.stream.synchronize()
        for st in states:
            st.close()
        self.states = []
        self.state = None
        self.dataset = None


class IID(_Baseline):
    """Uniform sampling of the unlabeled items; the best model has the lowest mean loss on the labels (iid.py)."""

    def __init__(self, dataset, loss_fn, *, gpus=None, shards=None, comm=None):
        self._setup(dataset, gpus, shards, comm)
        self.loss_fn = loss_fn
        self.stochastic = True
        self._risk_sum = torch.zeros(self.H, device=self.device)

    def _loss(self, col, true_class, dev):
        return self.loss_fn(col, torch.tensor([true_class], device=dev).expand(self.H))

    def get_next_item_to_label(self):
        self.stochastic = True
        n = len(self.d_u_idxs)
        idx = self.d_u_idxs[random.choice(range(n))]      # the same draw as random.choice over the list
        return idx, 1.0 / n

    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        # the per-label losses added in label order: the sum iid.py:37-43 recomputes from scratch
        # (a 16-bit slab's scores are widened first: the loss sees the fp32 values the reference loader would produce)
        self._risk_sum += self._label_losses(chosen_idx, true_class)

    def get_risk_estimates(self):
        risk = self._risk_sum.clone()
        if self.d_l_idxs:
            risk /= len(self.d_l_idxs)
        return risk

    def get_best_model_prediction(self):
        return self._min_risk_model(self.get_risk_estimates())


class Uncertainty(IID):
    """The unlabeled item of highest ensemble-mean entropy (uncertainty.py); a static score."""

    def __init__(self, dataset, loss_fn, *, gpus=None, shards=None, comm=None):
        super().__init__(dataset, loss_fn, gpus=gpus, shards=shards, comm=comm)
        for st in self.states:
            _hard, _dis, ens = st.scan(ens=True)
            with st._on():
                st.score = ensemble_entropy(ens, self.H)
            del _hard, _dis, ens
        self.stochastic = False

    def get_next_item_to_label(self):
        if not len(self.d_u_idxs):
            raise IndexError("max(): Expected reduction dim 0 to have non-zero size.")

        def draw_k(cnt):
            if cnt > 1:
                self.stochastic = True
                return int(torch.randperm(cnt)[0])
            return 0
        return self._select_extreme("score", True, draw_k)


class ActiveTesting(IID):
    """Kossen et al. (2021): items drawn with probability proportional to the expected loss under the ensemble-mean
    surrogate, summed over the models; risks by the LURE estimator (activetesting.py)."""

    _vma = False

    def __init__(self, dataset, loss_fn, *, gpus=None, shards=None, comm=None):
        super().__init__(dataset, loss_fn, gpus=gpus, shards=shards, comm=comm)
        for st in self.states:
            hard, _dis, ens = st.scan(ens=True)
            st.score = st.static_scores(hard, ens, vma=self._vma)
            del hard, _dis, ens
        self.M = 0
        self.losses = []
        self.qs = []
        self.stochastic = True

    def _loss(self, col, true_class, dev):
        return self.loss_fn(col, torch.tensor([true_class], device=dev).repeat(self.H), reduction="none")

    def _draw(self):
        total, n = self._total()
        if n == 0:
            raise IndexError("list index out of range")
        if not np.float32(total) > 0:                     # the normalised weights are 0 / 0
            raise ValueError("Total of weights must be finite")
        return self._weighted_draw(random.random())

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
        self.losses.append(self._label_losses(chosen_idx, true_class))
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
        total, n = self._total()
        if np.float32(total) < np.float32(1e-12):
            return self.d_u_idxs[random.choice(range(n))], 1.0 / n
        return self._weighted_draw(random.random())


class ModelPicker(_Baseline):
    """Karimi et al. (2021): the unlabeled item of least expected posterior entropy over the models, the best model
    the one with the most correct labels (modelpicker.py)."""

    def __init__(self, dataset, epsilon=0.46, *, gpus=None, shards=None, comm=None):
        self._setup(dataset, gpus, shards, comm)
        for st in self.states:
            st.hard, st.disagree, _ = st.scan(ens=False)
            with st._on():
                st.ent = torch.empty(st.N, dtype=torch.float32, device=st.dev)
                if self._xs:
                    st.post = torch.empty(self.H, dtype=torch.float32, device=st.dev)
                    st.row_in = torch.empty(self.H, dtype=torch.int16, device=st.dev)
        self._disagree_host = self._all_disagree()
        self._n_disagree = int(self._disagree_host.sum())     # unlabeled items some model disagrees on
        self.epsilon = float(epsilon)
        self.gamma = (1.0 - self.epsilon) / self.epsilon
        self.posterior = torch.ones(self.H, device=self.device) / self.H
        self.correct_counts = torch.zeros(self.H, dtype=torch.long, device=self.device)
        self.stochastic = True

    def _all_disagree(self):
        """The unanimity bits of ALL items on the host (one process per GPU: all-gathered from the ranks)."""
        parts = []
        for st in self.states:
            with st._on():
                parts.append(st.disagree.cpu().numpy())
        if not (self.group.world > 1 and len(self.states) == 1):
            return np.concatenate(parts)
        comm, st = self.group.comm, self.state
        with torch.cuda.device(st.dev):
            meta = comm.allgather(torch.tensor([st.n_offset, st.N], dtype=torch.int64, device=st.dev)).cpu().numpy()
            pad = torch.zeros(int(meta[:, 1].max()), dtype=torch.uint8, device=st.dev)
            pad[:st.N] = st.disagree
            allv = comm.allgather(pad).cpu().numpy()
        out = np.zeros(self.N, dtype=np.uint8)
        for r, (off, n) in enumerate(meta.tolist()):
            out[off:off + n] = allv[r, :n]
        return out

    def get_next_item_to_label(self):
        n = len(self.d_u_idxs)
        if n == 0:
            raise RuntimeError("min(): Expected reduction dim to be specified for input.numel() == 0.")
        for st in self.states:
            post = self.posterior
            if self._xs:                                      # this shard's replica of the posterior
                st.leave()
                with torch.cuda.device(st.dev):
                    st.post.copy_(self.posterior)
                st.enter()
                post = st.post
            with st._on():
                # gamma enters modelpicker.py:78 as a float32 factor
                st._call("coda_b200_mp_entropy", _ptr(st.hard), _ptr(post), self.H, st.N, self.C,
                         float(np.float32(self.gamma)), _ptr(st.labeled), _ptr(st.disagree), int(self._n_disagree > 0),
                         _ptr(st.ent), st._s())
        # drawn every step, one tie or many (modelpicker.py:70)
        idx, _val = self._select_extreme("ent", False, lambda cnt: int(torch.randint(cnt, (1,))[0]))
        return idx, 1.0 / float(n)

    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        if self._disagree_host[int(chosen_idx)]:
            self._n_disagree -= 1
        if self._xs:                                          # the owner's hard row, through the mailboxes
            preds = self._share(chosen_idx, lambda st, loc: st.hard[loc], "row_in").to(torch.int64) & 0xFFFF
        elif self.state.compact is not None:
            preds = self.state.hard[int(chosen_idx)].to(torch.int64) & 0xFFFF
        else:
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
