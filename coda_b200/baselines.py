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

Host-free loop: ``run_steps(k, labels, seed=...)`` runs ``k`` steps of main.py:91-94 (select, oracle, add_label,
best model) as one CUDA-graph replay per step and shard, with one host sync at the end; ``history()`` /
``best_history()`` read back the picks and per-step best models and bring the host-side state up to date, so API calls
and device loops can follow each other.  Draws whose consumption is known up front (IID's ``random.choice``, the
``random.random()`` of ActiveTesting and VMA) are made on the host before the loop with the API's own calls.  The
draws the reference makes from torch's generators (tie breaks, ModelPicker's draws) come from a Philox4x32-10 stream
by default, or with ``tie_rule="reference"`` from device replicas of torch's CPU and CUDA generators, call for call
(``include/coda_b200.h``, DESIGN.md §5b).

Checkpoints: ``state_dict()`` / ``load_state_dict()`` save and restore what a run has learned (labels, removed items,
the method's host-side sums, the loop history) and the three generators, with no layout; the next ``run_steps`` rebuilds
the device loop's sums from that host state (``_loop_upload``), so a resumed run continues bit for bit in one process.
"""
from __future__ import annotations

import bisect
import contextlib
import ctypes
import functools
import os
import random

import numpy as np
import torch

from . import _native as nat
from .base import ModelSelector
from .datasets import model_stride, walk
from .dist import ProcessGroup, default_comm, labels_per_device, shard_layout
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


HIST_CAP = 1 << 16          # device-loop history ring (slot = device-loop step % HIST_CAP), as CODA's
_LS_WORDS = 16              # loop words of coda_bl_loop_t (include/coda_b200.h)


def predraw(kind, k, n0):
    """The Python ``random`` draws of ``k`` steps, made with the calls the API path makes, in step order:
    ``kind = "choice"`` (IID, ``n0`` unlabeled items before the first step): ``random.choice(range(n0 - s))``;
    ``"random"`` (ActiveTesting, VMA): ``random.random()``; ``None``: nothing."""
    if kind == "choice":
        return [float(random.choice(range(n0 - s))) for s in range(k)]
    if kind == "random":
        return [random.random() for _ in range(k)]
    return []


def rewind(state, kind, j, n0):
    """Python ``random`` as after the first ``j`` steps' draws from ``state`` (the state before ``predraw``)."""
    random.setstate(state)
    predraw(kind, j, n0)


# torch.get_rng_state(): u64 seed, i32 left, i32 seeded, u64 next, then the 624 MT19937 words as u64 (low 32 bits),
# then the normal samplers' cache (5056 bytes in all)
_MT_WORDS = slice(24, 24 + 8 * 624)


def torch_rng_words(state: torch.Tensor) -> torch.Tensor:
    """torch.get_rng_state() -> the device replica's int32 [625]: the 624 words (as uint32 bits), then the position of
    the next word, 625 - left (torch draws ``if (--left == 0) twist; y = state[next++]``)."""
    b = state.numpy().tobytes()
    left = int(np.frombuffer(b, "<i4", 1, 8)[0])
    out = np.empty(625, np.uint32)
    out[:624] = np.frombuffer(b[_MT_WORDS], "<u8")
    out[624] = 625 - left
    return torch.from_numpy(out.view(np.int32))


def torch_rng_state(words: torch.Tensor, state0: torch.Tensor) -> torch.Tensor:
    """The inverse of ``torch_rng_words``: ``state0`` with its words, ``left`` and ``next`` taken from the replica and
    every other byte kept."""
    b = state0.numpy().copy()
    w = words.numpy().view(np.uint32)
    pos = int(w[624])
    b[8:12] = np.array([625 - pos], "<i4").view(np.uint8)
    b[16:24] = np.array([pos], "<u8").view(np.uint8)
    b[_MT_WORDS] = w[:624].astype("<u8").view(np.uint8)
    return torch.from_numpy(b)


def cuda_rng_words(state: torch.Tensor) -> torch.Tensor:
    """torch.cuda.get_rng_state() (u64 seed, i64 offset) -> the device replica's int64 [2]."""
    return torch.from_numpy(np.frombuffer(state.numpy().tobytes(), "<i8").copy())


def cuda_rng_state(words: torch.Tensor) -> torch.Tensor:
    return torch.from_numpy(words.numpy().astype("<i8").view(np.uint8).copy())


# -- checkpoints (state_dict / load_state_dict) ---------------------------------------------------------------------
STATE_VERSION = 1
# what each method (by its main.py --method name) has learned beyond the labels: the "fields" of its state
STATE_FIELDS = {"iid": ("risk_sum",), "uncertainty": ("risk_sum",), "activetesting": ("losses", "qs", "M"),
                "vma": ("losses", "qs", "M"), "model_picker": ("posterior", "correct_counts", "n_disagree")}
_HIST_KEYS = (("idx", torch.int64), ("q", torch.float64), ("tie", torch.int32), ("best", torch.int32),
              ("best_tie", torch.int32))
_STATE_KEYS = ("d_l_idxs", "d_l_ys", "removed", "stochastic", "dev_steps", "history", "fields", "rng")


def pack_state(method, H, N, C, epsilon=None, *, labeled=(), labels=(), removed=(), stochastic=False, history=None,
               fields=None, rng=None):
    """A competing selector's checkpoint from host values.  It holds ints, floats, strings, lists, tuples, dicts, None
    and CPU tensors only, so ``torch.save`` / ``torch.load`` (``weights_only=True``) round-trip it, and no shard layout.
    ``labeled`` / ``labels``: ``d_l_idxs`` / ``d_l_ys``; ``removed``: the items taken out of ``d_u_idxs`` without a label;
    ``history``: the device-loop arrays of ``history()`` / ``best_history()`` by key (idx, q, tie, best, best_tie;
    a missing key is empty); ``fields``: the method's own (``STATE_FIELDS``); ``rng``: ``{"python": random.getstate(),
    "torch": torch.get_rng_state(), "cuda": torch.cuda.get_rng_state(device)}``."""
    history = history or {}
    hist = {k: torch.tensor(np.asarray(history.get(k, ())), dtype=dt).reshape(-1) for k, dt in _HIST_KEYS}
    return {"version": STATE_VERSION, "method": method, "H": int(H), "N": int(N), "C": int(C),
            "epsilon": None if epsilon is None else float(epsilon),
            "d_l_idxs": [int(i) for i in labeled], "d_l_ys": [int(y) for y in labels],
            "removed": sorted(int(i) for i in removed), "stochastic": bool(stochastic),
            "dev_steps": int(hist["idx"].numel()), "history": hist, "fields": dict(fields or {}), "rng": dict(rng or {})}


def check_state(sd, method, H, N, C, epsilon=None):
    """Raise ``ValueError`` unless ``sd`` is a version-1 checkpoint of ``method`` on an (H, N, C) task (and, for
    ModelPicker, with this ``epsilon``) whose item lists and sums fit that task."""
    if not isinstance(sd, dict):
        raise ValueError(f"coda_b200.baselines: a state_dict is a dict, got {type(sd).__name__}")
    if sd.get("version") != STATE_VERSION:
        raise ValueError(f"coda_b200.baselines: state_dict version {sd.get('version')!r}; this package reads version "
                         f"{STATE_VERSION}")
    if sd.get("method") != method:
        raise ValueError(f"coda_b200.baselines: the state_dict is of method {sd.get('method')!r}, not {method!r}")
    if (sd.get("H"), sd.get("N"), sd.get("C")) != (H, N, C):
        raise ValueError(f"coda_b200.baselines: the state_dict belongs to a task of (H, N, C) = "
                         f"{(sd.get('H'), sd.get('N'), sd.get('C'))}, not {(H, N, C)}")
    eps = None if epsilon is None else float(epsilon)
    if sd.get("epsilon") != eps:
        raise ValueError(f"coda_b200.baselines: the state_dict has epsilon {sd.get('epsilon')!r}, this selector {eps!r}")
    missing = [k for k in _STATE_KEYS if k not in sd]
    missing += [k for k in STATE_FIELDS[method] if k not in (sd.get("fields") or {})]
    missing += [k for k, _ in _HIST_KEYS if k not in (sd.get("history") or {})]
    if missing:
        raise ValueError(f"coda_b200.baselines: the state_dict lacks {missing}")
    items = list(sd["d_l_idxs"]) + list(sd["removed"])
    if len(sd["d_l_ys"]) != len(sd["d_l_idxs"]) or len(set(items)) != len(items) or any(
            not 0 <= int(i) < N for i in items):
        raise ValueError("coda_b200.baselines: the state_dict's labeled and removed items are not distinct items of "
                         "the task with one label each")
    if any(int(sd["history"][k].numel()) != int(sd["dev_steps"]) for k, _ in _HIST_KEYS):
        raise ValueError("coda_b200.baselines: the state_dict's history arrays do not all hold dev_steps entries")
    f = sd["fields"]
    sizes = {"risk_sum": H, "posterior": H, "correct_counts": H}
    if any(k in f and f[k].numel() != n for k, n in sizes.items()) or (
            "losses" in f and (tuple(f["losses"].shape) != (int(f["M"]), H) or len(f["qs"]) != int(f["M"]))):
        raise ValueError(f"coda_b200.baselines: the state_dict's sums do not fit a task of H = {H} models")


def _synced(fn):
    """API calls after a device loop first bring the host-side state up to date (``history()``)."""
    @functools.wraps(fn)
    def call(self, *args, **kwargs):
        if self._loop_dirty:
            self.history()
        return fn(self, *args, **kwargs)
    return call


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

    def remove_marked(self, idx):
        """remove() of an item the device has already marked labeled."""
        idx = int(idx)
        if idx not in self:
            raise ValueError("list.remove(x): x not in list")
        self._removed.add(idx)
        bisect.insort(self._sorted, idx)

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
        from .datasets import CompactSlab, HostSlab
        self.compact = preds if isinstance(preds, CompactSlab) else None
        self.host = preds if isinstance(preds, HostSlab) else None       # streamed through the device by the scan
        if not ((isinstance(preds, torch.Tensor) or self.compact is not None or self.host is not None) and preds.is_cuda):
            raise NotImplementedError(_NO_CPU)
        H, N, C = (int(s) for s in preds.shape)
        if self.compact is not None:
            self.fmt = None
            self.model_stride = int(preds.ids.stride(0)) if H > 1 else N * preds.K
        elif self.host is not None:
            self.fmt = nat.slab_format(preds.dtype)
            self.model_stride = N * C
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
            else:                                          # a host slab in N-range chunks: the scan is per item
                walk(self.preds, lambda n0, n1, v: self._scan_dense(_ptr(v), model_stride(v), n1 - n0, _ptr(hard[n0:]),
                                                                    _ptr(pseudo[n0:]), _ptr(disagree[n0:]),
                                                                    _ptr(e[n0:]) if e is not None else None))
            flags = int(self.flags.item())
        if flags & nat.FLAG_NONFINITE_INPUT:
            raise RuntimeError("[NUMERIC ERROR] preds has bad values (NaN/Inf)")
        if flags & nat.FLAG_RANGE_INPUT:
            raise ValueError("coda_b200: dataset.preds must hold post-softmax scores in [0, 1] (coda/datasets.py:6)")
        return hard, disagree, e

    def _scan_dense(self, base, model_stride, n, hard, pseudo, disagree, e):
        H, C = self.H, self.C
        if self.fmt == nat.SLAB_F32:
            self._call("coda_b200_scan_slab", base, model_stride, H, n, C, hard, pseudo, disagree, e, _ptr(self.flags),
                       self._s())
        else:
            self._call("coda_b200_scan_slab_x", base, self.fmt, model_stride, H, n, C, hard, pseudo, disagree, e,
                       _ptr(self.flags), self._s())

    def column(self, loc):
        """The (H, C) fp32 scores of local item ``loc`` (a 16-bit slab widened, a compact slab densified)."""
        if self.compact is not None:
            return self.compact.item_column(loc)
        if self.host is not None:
            return self.host.item_column(loc)
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

    # -- the device loop (coda_b200_bl_* entry points) ------------------------------------------------------------
    def loop_alloc(self, method, n_global, gamma):
        """Loop words, per-method sums and history rings of this shard (once per selector)."""
        H = self.H
        with self._on():
            if getattr(self, "hard", None) is None:          # IID, Uncertainty, AT and VMA dropped their scan
                self.hard, self.disagree, _ = self.scan(ens=False)
            z = lambda *shape, dt: torch.zeros(shape, dtype=dt, device=self.dev)
            self.ls = z(_LS_WORDS, dt=torch.int64)
            self.pre = z(1, dt=torch.float64)
            self.counts = z(H, dt=torch.int32)
            lure = method in (nat.BL_ACTIVETESTING, nat.BL_VMA)
            self.s1, self.s2 = (z(H, dt=torch.float64), z(H, dt=torch.float64)) if lure else (None, None)
            self.lpost = z(H, dt=torch.float32) if method == nat.BL_MODELPICKER else None
            self.lzeros = z(self.N, dt=torch.float32) if method == nat.BL_IID else None
            self.h_idx = z(HIST_CAP, dt=torch.int64)
            self.h_q = z(HIST_CAP, dt=torch.float64)
            self.h_tie = z(HIST_CAP, dt=torch.int32)
            self.h_best = z(HIST_CAP, dt=torch.int32)
            self.h_btie = z(HIST_CAP, dt=torch.int32)
            self.h_loss = z(HIST_CAP, H, dt=torch.uint8) if lure else None
            self.trng = z(625, dt=torch.int32)                # tie_rule="reference": torch's CPU generator
            self.grng = z(2, dt=torch.int64)                  # and its CUDA generator (ModelPicker)
        self.lmethod, self.lgraph, self.lstruct = method, None, None
        self.lrule = "philox"
        self.lgamma_f32 = float(np.float32(gamma))            # gamma enters modelpicker.py:78 as a float32 factor
        self.n_global = int(n_global)
        # the vector the arg-extreme selection runs over (IID: all zeros, so the k-th tie is the k-th unlabeled item)
        self.lvec = {nat.BL_IID: self.lzeros, nat.BL_UNCERTAINTY: getattr(self, "score", None),
                     nat.BL_MODELPICKER: getattr(self, "ent", None)}.get(method)

    def loop_bind(self, labels, pre_len):
        """(Re)build the loop struct for these labels and a pre-draw buffer of at least ``pre_len``; a new struct
        drops the captured graph (its kernels hold the old pointers)."""
        if self.pre.numel() < pre_len:
            with self._on():
                self.pre = torch.zeros(max(pre_len, 2 * self.pre.numel()), dtype=torch.float64, device=self.dev)
            self.lstruct = None
        if self.lstruct is not None and self.lstruct.labels == labels.data_ptr():
            return
        a = nat.BlLoopStruct()
        a.method, a.H, a.N, a.n_offset, a.n_global = self.lmethod, self.H, self.N, self.n_offset, self.n_global
        a.hard, a.disagree, a.labeled, a.labels = _ptr(self.hard), _ptr(self.disagree), _ptr(self.labeled), _ptr(labels)
        a.pre, a.ls, a.best, a.total = _ptr(self.pre), _ptr(self.ls), _ptr(self.best), _ptr(self.total_buf)
        a.pick = _ptr(self.out)
        a.counts, a.s1, a.s2, a.post = _ptr(self.counts), _ptr(self.s1), _ptr(self.s2), _ptr(self.lpost)
        a.gamma = self.lgamma_f32
        a.hist_cap = HIST_CAP
        a.hist_idx, a.hist_q, a.hist_tie = _ptr(self.h_idx), _ptr(self.h_q), _ptr(self.h_tie)
        a.hist_best, a.hist_best_tie, a.hist_loss = _ptr(self.h_best), _ptr(self.h_btie), _ptr(self.h_loss)
        a.flags = _ptr(self.flags)
        self.lstruct, self.lgraph, self._labels_keep = a, None, labels

    def _lw(self, i):
        return self.ls.data_ptr() + 8 * i                     # address of loop word i

    def loop_rule(self, rule):
        """The tie rule of the next steps; the captured graph is of one rule."""
        if rule != self.lrule:
            self.lrule, self.lgraph = rule, None

    def loop_phase(self, phase):
        """Enqueue phase 0-3 of one device-loop step: the selection pass, the draw, the pick, the step kernel (with
        tie_rule="reference": the draw from torch's CPU generator, and the best model's tie redrawn after the step)."""
        m, a = self.lmethod, ctypes.byref(self.lstruct)
        lure = m in (nat.BL_ACTIVETESTING, nat.BL_VMA)
        ref = self.lrule == "reference"
        with self._on():
            if phase == 0:
                if lure:
                    self.total(self.score)
                    return
                if m == nat.BL_MODELPICKER:
                    self._call("coda_b200_mp_entropy_dev", _ptr(self.hard), _ptr(self.lpost), self.H, self.N, self.C,
                               self.lgamma_f32, _ptr(self.labeled), _ptr(self.disagree), self._lw(7), _ptr(self.ent),
                               self._s())
                self.extreme(self.lvec, m != nat.BL_MODELPICKER)
            elif phase == 1:
                if ref and m in (nat.BL_UNCERTAINTY, nat.BL_MODELPICKER):
                    self._call("coda_b200_bl_draw_ref", a, _ptr(self.trng), self._s())
                else:
                    self._call("coda_b200_bl_draw", a, self._s())
            elif phase == 2:
                if lure:
                    self._call("coda_b200_weighted_draw_xchg_dev", _ptr(self.score), _ptr(self.labeled), self.N,
                               _ptr(self.total_buf), self._lw(8), self._lw(2), self.n_offset, _ptr(self.part_f),
                               _ptr(self.out), self._x(), _ptr(self.flags), self._s())
                else:
                    self._call("coda_b200_select_kth_xchg_dev", _ptr(self.lvec), _ptr(self.labeled), self.N,
                               _ptr(self.part_i),
                               _ptr(self.best), self._lw(3), self._lw(2), self.n_offset, _ptr(self.out), self._x(),
                               _ptr(self.flags), self._s())
            else:
                self._call("coda_b200_bl_step", a, self._x(), self._s())
                if ref:
                    self._call("coda_b200_bl_best_ref", a, _ptr(self.trng), _ptr(self.grng), self._s())

    def loop_body(self):
        for phase in range(4):
            self.loop_phase(phase)

    def loop_capture(self):
        """Capture one step as a CUDA graph (nothing runs during the capture)."""
        torch.cuda.synchronize(self.dev)
        g = torch.cuda.CUDAGraph()
        cap = self.stream or torch.cuda.Stream(device=self.dev)
        with torch.cuda.device(self.dev):
            with torch.cuda.graph(g, stream=cap, capture_error_mode="relaxed"):
                self.loop_body()
        torch.cuda.synchronize(self.dev)
        self.lgraph = g

    def loop_replay(self):
        with self._on():
            if self.lgraph is None:
                self.loop_body()
            else:
                self.lgraph.replay()

    def read(self, t):
        """Host copy of ``t`` (a result of the calls above) as a list."""
        with self._on():
            return t.tolist()

    def timed_out(self):
        """True once an exchange of this shard gave up on a peer (the flag is sticky)."""
        with self._on():
            return bool(int(self.flags.item()) & nat.FLAG_XCHG_TIMEOUT)

    def close(self):
        self.lgraph = self.lstruct = self._labels_keep = None
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


def _default_pieces():
    """The competing selectors split a task into ``CODA_B200_GPUS`` pieces, else keep it whole."""
    env = os.environ.get("CODA_B200_GPUS")
    return max(1, int(env)) if env else 1


def _layout(dataset, gpus, shards, comm):
    """-> (group, [(shard slab, n_offset)] of this process) (``dist.shard_layout``)."""
    from .datasets import CompactSlab, HostSlab, PieceSlab
    preds = getattr(dataset, "preds", None)
    n_offset = int(getattr(dataset, "n_offset", 0))
    if not isinstance(preds, (HostSlab, PieceSlab)):         # one device slab: this rank's shard, or a task to split
        if not (isinstance(preds, (torch.Tensor, CompactSlab)) and preds.is_cuda):
            raise NotImplementedError(_NO_CPU)
        N = int(preds.shape[1])
        n_global = int(getattr(dataset, "n_global", N))
        if comm.world > 1:
            if gpus or shards:
                raise ValueError("coda_b200.baselines: gpus= / shards= split a task inside one process; under "
                                 "torch.distributed with world > 1 every rank is one shard (pass this rank's N-range)")
            _check_rank_ranges(preds, n_offset, N, n_global, comm)
        elif n_global != N:
            raise NotImplementedError("coda_b200.baselines: an N-range shard of a task needs its peers: run one "
                                      "process per shard under torch.distributed, or pass the whole task with gpus= / "
                                      "shards=")
    group, layout = shard_layout(preds, gpus, shards, comm, n_offset, default=_default_pieces)
    if not preds.is_cuda:                                    # pieces: after their own refusals
        raise NotImplementedError(_NO_CPU)
    return group, layout


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
        self._loop_dirty = False        # device-loop steps not yet mirrored into the host-side state
        self._loop_ready = False
        self._dev_steps = 0             # device-loop steps ever
        self._hist_seen = 0             # of which mirrored by history()
        self._dev_nlab = -1             # labels the device-side sums hold (-1: never written)
        self._hist = {k: [] for k in ("idx", "q", "tie", "best", "best_tie")}
        self._loop_labels = None

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

    # -- host-free loop ---------------------------------------------------------------------------------------------
    _loop_method = None             # nat.BL_* of the class
    _loop_draw = None               # predraw kind of the class

    def _loop_check(self, k, labels):
        from coda.options import accuracy_loss
        if isinstance(self.group, ProcessGroup):
            raise NotImplementedError("coda_b200.baselines: run_steps drives the shards of one process; with one "
                                      "process per GPU use the API loop, or gpus= / shards= in a single process")
        if getattr(self, "loss_fn", accuracy_loss) is not accuracy_loss:
            raise NotImplementedError("coda_b200.baselines: run_steps computes the loss on the device as "
                                      "hard[idx, h] != label (coda.options.accuracy_loss); use the API loop "
                                      "(get_next_item_to_label / add_label) for another loss_fn")
        if not isinstance(labels, torch.Tensor) or labels.dim() != 1 or labels.numel() != self.N:
            raise ValueError(f"coda_b200.baselines: labels must be a 1-d tensor of all {self.N} labels")
        left = len(self.d_u_idxs) - (self._dev_steps - self._hist_seen)
        if not 0 <= k <= left:
            raise ValueError(f"coda_b200.baselines: run_steps({k}) with {left} unlabeled items left")

    def _loop_bind_labels(self, labels):
        if self._loop_labels is None or self._loop_labels[0] is not labels:
            self._loop_labels = (labels, labels_per_device(labels, [st.dev for st in self.states]))
        return self._loop_labels[1]

    def _loop_upload(self, seed):
        """Write the host-side state (labels so far, the method's sums) into every shard's loop buffers."""
        m, H, nlab = self._loop_method, self.H, len(self.d_l_idxs)
        words = torch.zeros(_LS_WORDS, dtype=torch.int64)
        words[0], words[5], words[6] = nlab, self._dev_steps, seed
        sums = {}                                      # staged on the host: no shard stream reads the caller's tensors
        if m in (nat.BL_IID, nat.BL_UNCERTAINTY):
            sums["counts"] = self._risk_sum.round().to(torch.int32).cpu()
        elif m == nat.BL_MODELPICKER:
            words[7] = int(self._n_disagree)
            sums["counts"] = self.correct_counts.to(torch.int32).cpu()
            sums["lpost"] = self.posterior.cpu()
        else:                                        # the LURE sums, in the order bl_step adds them
            s1, s2 = np.zeros(H), np.zeros(H)
            Ng = float(self.N)
            for mm, (L, q) in enumerate(zip(self.losses, self.qs), start=1):
                L = L.reshape(-1).double().cpu().numpy() != 0
                a = 1.0 / ((Ng - mm + 1.0) * float(q)) - 1.0
                t = a / (Ng - mm) if Ng - mm > 0 else 0.0
                s1 = s1 + np.where(L, 1.0, 0.0)
                s2 = s2 + np.where(L, t, 0.0)
            sums["s1"], sums["s2"] = torch.from_numpy(s1), torch.from_numpy(s2)
        for st in self.states:
            st.enter()
            with st._on():
                st.ls.copy_(words)
                for name, v in sums.items():
                    getattr(st, name).copy_(v)
        self._dev_nlab = nlab

    def _reference_refusals(self):
        if self._loop_method == nat.BL_UNCERTAINTY and self.N >= nat.RANDPERM32_MAX:
            raise NotImplementedError(f"coda_b200.baselines: tie_rule='reference' mirrors torch.randperm's 32-bit "
                                      f"branch, which takes fewer than {nat.RANDPERM32_MAX} items; got {self.N}")

    def _rng_upload(self):
        """tie_rule="reference": torch's CPU generator (and for ModelPicker the CUDA generator of the dataset's
        device) -> every shard's replicas; returns what ``_rng_download`` needs."""
        cpu = torch.get_rng_state()
        if cpu.numel() != 5056:
            raise RuntimeError(f"coda_b200.baselines: torch.get_rng_state() has {cpu.numel()} bytes, the replica "
                               f"reads the layout of 5056")
        gpu = torch.cuda.get_rng_state(self.device) if self._loop_method == nat.BL_MODELPICKER else None
        if gpu is not None and gpu.numel() != 16:
            raise RuntimeError(f"coda_b200.baselines: torch.cuda.get_rng_state() has {gpu.numel()} bytes, the replica "
                               f"reads {{seed, offset}} (16)")
        words = torch_rng_words(cpu)
        gw = cuda_rng_words(gpu) if gpu is not None else None
        for st in self.states:
            st.enter()
            with st._on():
                st.trng.copy_(words)
                if gw is not None:
                    st.grng.copy_(gw)
        return cpu, words, gw

    def _rng_download(self, up):
        """The replicas -> torch's generators (only the words and the position or offset change); raises if the
        shards' replicas differ."""
        cpu, words, gw = up
        got = []
        for st in self.states:
            with st._on():
                got.append((st.trng.cpu(), st.grng.cpu()))
        t, g = got[0]
        if any(not torch.equal(t2, t) or (gw is not None and not torch.equal(g2, g)) for t2, g2 in got[1:]):
            raise RuntimeError("coda_b200.baselines: the shards' replicas of torch's generators differ after run_steps")
        if not torch.equal(t, words):                  # untouched: keep torch's own bytes (e.g. left = 1, next = 0)
            torch.set_rng_state(torch_rng_state(t, cpu))
        if gw is not None and not torch.equal(g, gw):
            torch.cuda.set_rng_state(cuda_rng_state(g), self.device)

    def run_steps(self, k, labels, *, seed=None, tie_rule="philox"):
        """``k`` steps of main.py:91-94 (get_next_item_to_label, oracle, add_label, get_best_model_prediction) on the
        device: after a warm-up step, one CUDA-graph replay per step and shard (``CODA_B200_GRAPH=0``: the same
        kernels launched one by one), one host sync at the end.  ``labels``: int64 tensor of all N labels (cached per
        device).  Python ``random`` is consumed as by ``k`` API steps.  When a step needs what the device loop does
        not do (VMA's uniform fallback, ActiveTesting's zero total), the remaining steps run on the API path, with the
        API's result or error.  Returns the number of steps performed (``k``); read ``history()`` /
        ``best_history()`` afterwards.

        ``tie_rule``: where the draws the reference makes from torch's generators come from (Uncertainty's item ties,
        ModelPicker's item and best model, the best-model ties of the others).  ``"philox"`` (the default): a
        Philox4x32-10 stream keyed by ``seed`` (``None``: one ``torch.randint`` on the CPU generator), the same
        distribution as the reference's.  ``"reference"``: the same draws, from device replicas of torch's CPU
        generator and of the CUDA generator of the dataset's device, written back afterwards, so the picks, best
        models and ``torch.get_rng_state()`` / ``torch.cuda.get_rng_state()`` are those of ``k`` API steps.  It takes
        no ``seed``."""
        if tie_rule not in ("philox", "reference"):
            raise ValueError(f"tie_rule must be 'philox' or 'reference', got {tie_rule!r}")
        ref = tie_rule == "reference"
        if ref and seed is not None:
            raise ValueError("coda_b200.baselines: seed= keys the Philox stream of tie_rule='philox'; "
                             "tie_rule='reference' draws from torch's generators")
        k = int(k)
        self._loop_check(k, labels)
        if ref:
            self._reference_refusals()
        if k == 0:
            return 0
        per_dev = self._loop_bind_labels(labels)
        if ref:
            seed = 0
        elif seed is None:
            seed = int(torch.randint(0, 1 << 62, (1,)).item())
        seed = int(seed) & ((1 << 64) - 1)
        seed = seed - (1 << 64) if seed >= 1 << 63 else seed
        if not self._loop_ready:
            gamma = getattr(self, "gamma", 1.0)
            for st in self.states:
                st.loop_alloc(self._loop_method, self.N, gamma)
            self._loop_ready = True
        n0 = len(self.d_u_idxs) - (self._dev_steps - self._hist_seen)
        state0 = random.getstate()
        pre = predraw(self._loop_draw, k, n0)
        pre_host = torch.tensor(pre or [0.0], dtype=torch.float64).pin_memory()
        for st in self.states:
            st.enter()                                # after what the caller's stream enqueued (API-path state)
            st.loop_bind(per_dev[st.dev], k)
            st.loop_rule(tie_rule)
        if not self._loop_dirty and self._dev_nlab != len(self.d_l_idxs):
            self._loop_upload(seed)
        up = self._rng_upload() if ref else None
        for st in self.states:
            with st._on():
                st.pre[:pre_host.numel()].copy_(pre_host, non_blocking=True)
                st.ls[1:3].zero_()
                st.ls[6].fill_(seed)
        use_graph = os.environ.get("CODA_B200_GRAPH", "1") != "0"
        done_before = self._dev_steps
        left = k
        while left:
            if self._dev_steps - self._hist_seen >= HIST_CAP:
                self._pull()                          # the ring is full: mirror it before it wraps
            n = min(left, HIST_CAP - (self._dev_steps - self._hist_seen))
            j = 0
            if use_graph and any(st.lgraph is None for st in self.states):
                for phase in range(4):                # warm-up, in lock-step phases over the shards: a kernel's first
                    for st in self.states:            # launch may load its module while a peer's exchange spins
                        st.loop_phase(phase)
                for st in self.states:
                    st.loop_capture()
                j = 1
            for _ in range(n - j):
                if use_graph:
                    for st in self.states:
                        st.loop_replay()
                else:
                    for phase in range(4):
                        for st in self.states:
                            st.loop_phase(phase)
            left -= n
            self._dev_steps += n                      # provisional; corrected from the device below
            self._loop_dirty = True
        with self.state._on():
            done = int(self.state.ls[1].item())
        self._check_exchanges()
        self._dev_steps = done_before + done
        self._dev_nlab = len(self.d_l_idxs) + (self._dev_steps - self._hist_seen)
        self._loop_dirty = self._dev_steps > self._hist_seen
        if ref:
            self._rng_download(up)
        if done < k:                                   # the API path takes over where the device loop stopped
            self.history()
            rewind(state0, self._loop_draw, done, n0)
            lab = self._loop_labels[0]
            for _ in range(k - done):
                idx, q = self.get_next_item_to_label()
                self.add_label(idx, int(lab[idx]), q)
                self.get_best_model_prediction()
        return k

    def _pull(self):
        """Mirror the device-loop steps not yet seen into the host-side state."""
        st = self.state
        with st._on():
            ls = st.ls.cpu().tolist()
        n0, n1 = self._hist_seen, int(ls[5])                # ls[5]: device-loop steps ever
        self._dev_steps = n1
        if n1 <= n0:
            self._loop_dirty = False
            return
        with st._on():
            slots = torch.arange(n0, n1, device=st.dev) % HIST_CAP
            got = {k: getattr(st, "h_" + k)[slots].cpu().numpy() for k in ("idx", "q", "tie", "best", "btie")}
            loss = st.h_loss[slots].to(torch.float32) if st.h_loss is not None else None
        self._check_exchanges()
        idx = got["idx"].astype(np.int64)
        lab = self._loop_labels[0]
        ys = lab[torch.as_tensor(idx, device=lab.device)].cpu().tolist() if lab.is_cuda else lab[idx].tolist()
        for i, y in zip(idx.tolist(), ys):
            self.d_u_idxs.remove_marked(i)
            self.d_l_idxs.append(int(i))
            self.d_l_ys.append(int(y))
        for key, v in (("idx", idx), ("q", got["q"]), ("tie", got["tie"]), ("best", got["best"]),
                       ("best_tie", got["btie"])):
            self._hist[key].append(v)
        m = self._loop_method
        with st._on():
            if m in (nat.BL_IID, nat.BL_UNCERTAINTY):
                self._risk_sum = st.counts.to(torch.float32)
            elif m == nat.BL_MODELPICKER:
                self.posterior = st.lpost.clone()
                self.correct_counts = st.counts.to(torch.int64)
                self._n_disagree = int(ls[7])
            else:
                self.losses.extend(loss.unbind(0))
                self.qs.extend(float(q) for q in got["q"])
                self.M += n1 - n0
        if got["tie"].any() or got["btie"].any():
            self.stochastic = True
        st.leave()                                     # the caller's stream reads what shard 0's stream produced
        self._hist_seen = n1
        self._dev_nlab = len(self.d_l_idxs)
        self._loop_dirty = False

    def _hist_arrays(self, *keys):
        out = []
        for key in keys:
            parts = self._hist[key]
            out.append(np.concatenate(parts) if parts else np.zeros(0, np.float64 if key == "q" else np.int64))
        return tuple(out)

    def history(self):
        """(idx, q, tie) of every device-loop step so far (``tie[s] = 1``: the item was drawn among exactly tied items);
        also brings the host-side state (``d_l_idxs``, ``d_l_ys``, ``d_u_idxs``, the method's sums, ``stochastic``) up
        to date."""
        if self._loop_dirty:
            self._pull()
        return self._hist_arrays("idx", "q", "tie")

    def best_history(self):
        """(best, best_tie) of every device-loop step: the model ``get_best_model_prediction()`` would have returned
        after that step, and 1 where it was drawn among exactly tied models."""
        if self._loop_dirty:
            self._pull()
        return self._hist_arrays("best", "best_tie")

    # -- checkpoint / resume (the reference restarts a killed seed from step 0) -------------------------------------
    _state_method = None            # the method's name in its state dict (main.py --method)

    def _state_refusals(self):
        if self.group.world > 1 and len(self.states) == 1:
            raise NotImplementedError("coda_b200.baselines: state_dict / load_state_dict need all items in one "
                                      "process: build the selector with gpus= / shards= (one process driving all "
                                      "GPUs) instead of one process per GPU")

    def state_dict(self):
        """The run so far as a plain dict (``pack_state``): the labels, the items removed without one, the method's
        sums, ``stochastic``, the device-loop history and the states of Python ``random``, torch's CPU generator and
        the CUDA generator of the dataset's device.  Device-loop steps not yet mirrored are pulled first.  It holds
        no layout: a selector of the same method on the same slab values loads it under any shard layout, slab width
        or piece split."""
        self._state_refusals()
        if self._loop_dirty:
            self._pull()
        labeled = set(self.d_l_idxs)
        keys = [k for k, _ in _HIST_KEYS]
        rng = {"python": random.getstate(), "torch": torch.get_rng_state(),
               "cuda": torch.cuda.get_rng_state(self.device)}
        return pack_state(self._state_method, self.H, self.N, self.C, getattr(self, "epsilon", None),
                          labeled=self.d_l_idxs, labels=self.d_l_ys,
                          removed=[i for i in self.d_u_idxs._removed if i not in labeled], stochastic=self.stochastic,
                          history=dict(zip(keys, self._hist_arrays(*keys))), fields=self._state_fields(), rng=rng)

    def load_state_dict(self, sd, restore_rng=True):
        """Resume a run saved by ``state_dict`` on a freshly built selector of the same method on the same task: the
        next API steps and ``run_steps`` continue it bit for bit.  Every shard's labeled mask is rebuilt from the item
        lists, and the device loop is re-uploaded from the restored host state on the next ``run_steps``.
        ``restore_rng=False`` leaves the caller's generators as they are."""
        self._state_refusals()
        check_state(sd, self._state_method, self.H, self.N, self.C, getattr(self, "epsilon", None))
        items = [int(i) for i in sd["d_l_idxs"]] + [int(i) for i in sd["removed"]]
        for st in self.states:
            st.enter()
            loc = [i - st.n_offset for i in items if 0 <= i - st.n_offset < st.N]
            with st._on():
                st.labeled.zero_()
                if loc:
                    st.labeled[torch.tensor(loc, dtype=torch.int64, device=st.dev)] = 1
            st.leave()
            st.lgraph = None                                   # captured graphs and loop words are of the old run
        self.d_u_idxs._removed = set(items)
        self.d_u_idxs._sorted = sorted(items)
        self.d_l_idxs = [int(i) for i in sd["d_l_idxs"]]
        self.d_l_ys = [int(y) for y in sd["d_l_ys"]]
        self.stochastic = bool(sd["stochastic"])
        h = sd["history"]
        self._hist = {k: [h[k].numpy().copy()] if h[k].numel() else [] for k, _ in _HIST_KEYS}
        self._dev_steps = self._hist_seen = int(sd["dev_steps"])
        self._loop_dirty = False
        self._dev_nlab = -1                                    # the next run_steps uploads the restored sums
        self._load_fields(sd["fields"])
        if restore_rng:
            rng = sd["rng"]
            random.setstate(rng["python"])
            torch.set_rng_state(rng["torch"])
            torch.cuda.set_rng_state(rng["cuda"], self.device)

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

    _loop_method, _loop_draw = nat.BL_IID, "choice"
    _state_method = "iid"

    def __init__(self, dataset, loss_fn, *, gpus=None, shards=None, comm=None):
        self._setup(dataset, gpus, shards, comm)
        self.loss_fn = loss_fn
        self.stochastic = True
        self._risk_sum = torch.zeros(self.H, device=self.device)

    def _state_fields(self):
        return {"risk_sum": self._risk_sum.cpu()}

    def _load_fields(self, f):
        self._risk_sum = f["risk_sum"].to(self.device, torch.float32)

    def _loss(self, col, true_class, dev):
        return self.loss_fn(col, torch.tensor([true_class], device=dev).expand(self.H))

    @_synced
    def get_next_item_to_label(self):
        self.stochastic = True
        n = len(self.d_u_idxs)
        idx = self.d_u_idxs[random.choice(range(n))]      # the same draw as random.choice over the list
        return idx, 1.0 / n

    @_synced
    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        # the per-label losses added in label order: the sum iid.py:37-43 recomputes from scratch
        # (a 16-bit slab's scores are widened first: the loss sees the fp32 values the reference loader would produce)
        self._risk_sum += self._label_losses(chosen_idx, true_class)

    @_synced
    def get_risk_estimates(self):
        risk = self._risk_sum.clone()
        if self.d_l_idxs:
            risk /= len(self.d_l_idxs)
        return risk

    @_synced
    def get_best_model_prediction(self):
        return self._min_risk_model(self.get_risk_estimates())


class Uncertainty(IID):
    """The unlabeled item of highest ensemble-mean entropy (uncertainty.py); a static score."""

    _loop_method, _loop_draw = nat.BL_UNCERTAINTY, None
    _state_method = "uncertainty"

    def __init__(self, dataset, loss_fn, *, gpus=None, shards=None, comm=None):
        super().__init__(dataset, loss_fn, gpus=gpus, shards=shards, comm=comm)
        for st in self.states:
            _hard, _dis, ens = st.scan(ens=True)
            with st._on():
                st.score = ensemble_entropy(ens, self.H)
            del _hard, _dis, ens
        self.stochastic = False

    @_synced
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
    _loop_method, _loop_draw = nat.BL_ACTIVETESTING, "random"
    _state_method = "activetesting"

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

    def _state_fields(self):
        # one [H] row per label (get_lure_risks_and_vars stacks and views them as [H][M] whatever their shape)
        losses = torch.stack([L.reshape(-1) for L in self.losses]).cpu() if self.losses else torch.zeros(0, self.H)
        return {"losses": losses, "qs": [float(q) for q in self.qs], "M": int(self.M)}

    def _load_fields(self, f):
        self.losses = list(f["losses"].to(self.device).unbind(0))
        self.qs = [float(q) for q in f["qs"]]
        self.M = int(f["M"])

    def _loss(self, col, true_class, dev):
        return self.loss_fn(col, torch.tensor([true_class], device=dev).repeat(self.H), reduction="none")

    def _draw(self):
        total, n = self._total()
        if n == 0:
            raise IndexError("list index out of range")
        if not np.float32(total) > 0:                     # the normalised weights are 0 / 0
            raise ValueError("Total of weights must be finite")
        return self._weighted_draw(random.random())

    @_synced
    def get_next_item_to_label(self):
        return self._draw()

    def get_vs(self):
        """LURE weights v_m (Farquhar et al. 2021) of the labels so far, m = 1 .. M."""
        N, M = self.N, self.M
        return [1 + ((N - M) / (N - m)) * (1 / ((N - m + 1) * q) - 1) for m, q in enumerate(self.qs, start=1)]

    @_synced
    def get_lure_risks_and_vars(self):
        losses = torch.stack(self.losses, dim=1).view(self.H, -1)
        weighted = torch.tensor(self.get_vs(), device=self.device).unsqueeze(0) * losses
        return weighted.mean(dim=1), weighted.var(dim=1, unbiased=True) / self.M

    @_synced
    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        self.losses.append(self._label_losses(chosen_idx, true_class))
        self.qs.append(selection_prob)
        self.M += 1

    @_synced
    def get_risk_estimates(self):
        return self.get_lure_risks_and_vars()[0]

    @_synced
    def get_best_model_prediction(self):
        if self.losses:
            return self._min_risk_model(self.get_risk_estimates())
        return torch.arange(self.H, device=self.device)[random.choice(range(self.H))]


class VMA(ActiveTesting):
    """Matsuura & Hara (2023): items drawn with probability proportional to sum_{h < h'} |loss_h - loss_h'| under the
    ensemble-mean surrogate (vma.py); uniform when every score is 0."""

    _vma = True
    _loop_method = nat.BL_VMA
    _state_method = "vma"

    @_synced
    def get_next_item_to_label(self):
        total, n = self._total()
        if np.float32(total) < np.float32(1e-12):
            return self.d_u_idxs[random.choice(range(n))], 1.0 / n
        return self._weighted_draw(random.random())


class ModelPicker(_Baseline):
    """Karimi et al. (2021): the unlabeled item of least expected posterior entropy over the models, the best model
    the one with the most correct labels (modelpicker.py)."""

    _loop_method = nat.BL_MODELPICKER
    _state_method = "model_picker"

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

    def _state_fields(self):
        return {"posterior": self.posterior.cpu(), "correct_counts": self.correct_counts.cpu(),
                "n_disagree": int(self._n_disagree)}

    def _load_fields(self, f):
        self.posterior = f["posterior"].to(self.device, torch.float32)
        self.correct_counts = f["correct_counts"].to(self.device, torch.int64)
        self._n_disagree = int(f["n_disagree"])

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

    @_synced
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

    @_synced
    def add_label(self, chosen_idx, true_class, selection_prob=None):
        self._record(chosen_idx, true_class)
        if self._disagree_host[int(chosen_idx)]:
            self._n_disagree -= 1
        if self._xs:                                          # the owner's hard row, through the mailboxes
            preds = self._share(chosen_idx, lambda st, loc: st.hard[loc], "row_in").to(torch.int64) & 0xFFFF
        elif self.state.compact is not None:
            preds = self.state.hard[int(chosen_idx)].to(torch.int64) & 0xFFFF
        else:
            st = self.state                                   # the one shard's slab (a ShardedSlab's only piece)
            preds = st.column(int(chosen_idx) - st.n_offset).argmax(dim=1)
        self.correct_counts += (preds == true_class).long()
        self.posterior = self.update_posterior(self.posterior, preds, true_class, self.gamma)

    def update_posterior(self, posterior, predictions_i, oracle_i, gamma):
        post = posterior * (gamma ** (predictions_i == oracle_i).float())
        return post / post.sum()

    @_synced
    def get_best_model_prediction(self):
        if not self.d_l_idxs:
            return torch.randint(self.H, (1,), device=self.device).item()
        ties = torch.nonzero(self.correct_counts == torch.max(self.correct_counts)).flatten()
        return ties[torch.randint(len(ties), (1,), device=self.device)].item()


from .eps_search import eps_search_run_key, modelpicker_eps_search  # noqa: E402  (uses _DeviceState above)

__all__ = ["IID", "Uncertainty", "ActiveTesting", "VMA", "ModelPicker", "ensemble_entropy", "modelpicker_eps_search",
           "eps_search_run_key"]
