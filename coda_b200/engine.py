"""Device-side state and kernel sequencing for one shard of the CODA acquisition path.

PyTorch is used for device memory, streams, CUDA graphs and the construction-time all-reduce -- the arithmetic of
the hot path and the per-step exchanges between shards are in the C-ABI library (``include/coda_b200.h``).

Modes (what is kept between steps; results are the same):
  ``incremental``   the normalised P(best | hypothetical) row of every row is cached; a label of
                    class t only invalidates the rows of class t (coda.py:317 touches row t only)
                    and the marginal refresh is the rank-1 column update of coda.py:319.
  ``recompute``     every step recomputes all rows from the tables (no row cache).
  ``recompute_all`` additionally rebuilds all class tables and re-runs the full slab pass of
                    ``update_pi_hat`` every step -- the reference's literal per-step work.

One acquisition step on the device (host-free loop, ``CODA.run_steps``; everything below is ONE CUDA graph):

    step_select   merge block records, exchange with the peers, arg-max, label lookup, D[h][t][p_h] += lr, gather list
    ---- fork ----  side stream: beta_tables(class t) -> pair_rows(class t)        main: pi_rank1 (marginal refresh)
    step_mixture  exchange the marginal sums, pi_hat, P(best), H_before, argmax         (needs PB[t] from the side)
    ---- join ----
    row_gains + gain_eig        the scoring pass for the NEXT selection -> block records
"""
from __future__ import annotations

import contextlib
import math
import os

import numpy as np
import torch

from . import _native as nat
from .datasets import model_stride, walk

_CONST_SLOTS = {}          # device index -> set of constant-memory term-table slots in use (csrc/slab.cu c_terms_bank)
_CONST_TERMS = 3584


def _acquire_const_slot(dev_index, H):
    per = (2 * H + 63) // 64 * 64
    used = _CONST_SLOTS.setdefault(dev_index, set())
    for s in range(_CONST_TERMS // per):
        if s not in used:
            used.add(s)
            return s
    return -1                  # every slot of this device is taken: the shared-memory copy of the list is used


def _release_const_slot(dev_index, slot):
    if slot is not None and slot >= 0:
        _CONST_SLOTS.get(dev_index, set()).discard(slot)


TIE_CAP = 256
REP_WORDS = 12 + TIE_CAP + TIE_CAP // 2     # [flags | record (8) | tie hdr (2) | pad | tie idx | tie val]
MODES = ("incremental", "recompute", "recompute_all")
TABLE_BATCH_BYTES = 512 << 20
HIST_CAP = 1 << 16
# With prefilter_n = m the engine scores only the sample when m * PREFILTER_ROW_COST_RATIO <= N.  Fitted by
# tools/bench_prefilter.py on an H100 80GB HBM3 at 700 W, cfg3 (256 x 5e5 x 100): the sampled pass takes
# 0.116 ms + 0.032 us per item (m = 1 000 ... 125 000), the full pass 0.885 ms, so they cross at m = 24 050 = N / 20.8
# (BASELINE.md §6b).
PREFILTER_ROW_COST_RATIO = 20.8
PREFILTER_SCORING = ("auto", "sample", "full")


def _ptr(t):
    return t.data_ptr() if t is not None else None


class _PinnedHost:
    """A host tensor page-locked and mapped for the device at its own address (coda_b200_host_register) for as long as
    this object lives: the host shadow slots of a host-resident slab."""

    def __init__(self, shape, dtype, lib):
        nbytes = math.prod(shape) * torch.empty(0, dtype=dtype).element_size()
        try:
            self.t = torch.empty(shape, dtype=dtype)
        except RuntimeError as e:
            raise MemoryError(f"coda_b200: cannot allocate {nbytes} bytes of host memory for the host shadow slots "
                              f"{tuple(shape)}: {e}") from e
        self.lib = lib
        if lib.coda_b200_host_register(self.t.data_ptr(), nbytes) != nat.OK:
            msg = nat.last_error()
            self.t = None
            raise MemoryError(f"coda_b200: cannot page-lock {nbytes} bytes of host memory for the host shadow slots "
                              f"{tuple(shape)}: {msg}")

    def data_ptr(self):
        return self.t.data_ptr()

    def __del__(self):
        if getattr(self, "t", None) is not None:
            self.lib.coda_b200_host_unregister(self.t.data_ptr())
            self.t = None


def shadow_slots(free: int, reserve: int, slot_bytes: int, want: int, ens: bool, left: int = 1, total: int = 1,
                 ens_slot_bytes: int | None = None):
    """-> (model slots, ensemble slots) of one shard's shadow.  ``free``: device bytes free now; ``total`` shards on
    the device keep ``reserve`` bytes each, and the ``left`` shards still to be sized (this one included) split the rest
    equally.  The ensemble slot (one per step, in every list with the majority shortcut) comes first, then up to
    ``want`` models.  ``slot_bytes``: one model slot (the slab's element size); ``ens_slot_bytes``: the ensemble slot,
    which is fp32 (default: ``slot_bytes``)."""
    share = max(0, (free - total * reserve) // max(1, left))
    eb = slot_bytes if ens_slot_bytes is None else ens_slot_bytes
    ne = 1 if ens and share >= eb else 0
    return int(max(0, min(want, (share - ne * eb) // slot_bytes))), ne


class Engine:
    rep_words = REP_WORDS

    def __init__(self, preds: torch.Tensor, *, alpha: float, learning_rate: float, multiplier: float,
                 uniform_prior: bool, hyp_w: float = 1.0, mode: str = "incremental", n_offset: int = 0,
                 n_global: int | None = None, world: int = 1, own_stream: bool = False, prefilter_n: int = 0,
                 q: str = "eig"):
        from .datasets import CompactSlab, HostSlab
        if mode not in MODES:
            raise ValueError(f"mode must be one of {MODES}")
        self.compact = preds if isinstance(preds, CompactSlab) else None
        # a host-resident slab: streamed through the device for construction, every model in a shadow slot afterwards
        self.host = preds if isinstance(preds, HostSlab) else None
        if not ((isinstance(preds, torch.Tensor) or self.compact is not None or self.host is not None) and preds.is_cuda):
            raise RuntimeError("coda_b200: dataset.preds must live on a CUDA (sm_90a) device; "
                               "there is no CPU path in this package")
        H, N, Cc = (int(s) for s in preds.shape)
        if N < 1:
            raise ValueError("coda_b200: empty shard (fewer items than shards?)")
        if self.compact is not None:
            if mode == "recompute_all":
                raise NotImplementedError("coda_b200: mode='recompute_all' is not offered for a compact slab")
            self.K = self.compact.K
        elif self.host is not None:
            if mode == "recompute_all":
                raise NotImplementedError("coda_b200: mode='recompute_all' re-reads the whole slab every step; it is not "
                                          "offered for a host-resident slab")
        else:
            nat.slab_format(preds.dtype)          # float32, float16 or bfloat16, else TypeError
            if preds.dim() != 3:
                raise TypeError("coda_b200: preds must be an (H, N, C) tensor (coda/datasets.py:14)")
            if not (preds.stride(2) == 1 and preds.stride(1) == Cc and (H == 1 or preds.stride(0) >= N * Cc)):
                raise ValueError("coda_b200: preds must be (H, N, C) with contiguous items (an N-range view of a "
                                 "contiguous slab is fine)")
        self.lib = nat.load()
        self.preds = preds
        # slab element type: a 16-bit slab is read at its stored width and widened to fp32 in every kernel
        self.fmt = nat.slab_format(preds.dtype) if self.compact is None else nat.SLAB_F32
        self.esz = int(preds.element_size()) if self.compact is None else 4
        self.kernels = {}                                     # construction kernels that ran (see _record_kernels)
        self.dev = preds.device
        with torch.cuda.device(self.dev):
            nat.require_device()
            # sector gathers of the rank-1 refresh: ask for 64-byte L2 fills (the default 128 doubles their DRAM
            # traffic; streaming kernels measured the same at 64 and 128).  A per-device limit.
            nat.check(self.lib.coda_b200_set_l2_fetch_granularity(int(os.environ.get("CODA_B200_L2_FETCH", "64"))), "l2_fetch")
        self.H, self.N, self.C = H, N, Cc
        if self.compact is not None:
            self.model_stride = int(self.compact.ids.stride(0)) if H > 1 else N * self.K     # elements of ids / probs
        elif self.host is not None:
            self.model_stride = N * Cc                        # each chunk the slab streams through is contiguous
        else:
            self.model_stride = int(preds.stride(0)) if H > 1 else N * Cc
        self.Hp = (H + 31) // 32 * 32
        self.W = self.Hp // 32
        self.P = 256
        self.T = Cc * (1 + H)
        self.mode = mode
        self.world = int(world)
        self.n_offset = int(n_offset)
        self.n_global = int(n_global if n_global is not None else N)
        self.lr = float(learning_rate)
        self.hyp_w = float(hyp_w)
        self.prior_strength = 1 - alpha                       # coda.py:189
        self.multiplier = float(multiplier)
        self.uniform_prior = bool(uniform_prior)
        if H > 1024:
            raise NotImplementedError("coda_b200: H > 1024 models is not supported yet")
        if Cc > 4096:
            raise NotImplementedError("coda_b200: C > 4096 classes is not supported yet")
        self.fx_shift = max(8, min(40, 62 - math.ceil(math.log2(self.n_global + 1))))
        self.counters = {"launches": 0}
        # CODA_B200_OVERLAP=0: class-t table / row refresh on the main stream instead of a side stream
        self.overlap = os.environ.get("CODA_B200_OVERLAP", "1") != "0"
        self.use_graph = os.environ.get("CODA_B200_GRAPH", "1") != "0"
        # prefilter_n: score only the sampled items each step (see _choose_sample_scoring)
        self.pf_m = int(prefilter_n or 0) if q == "eig" else 0
        self.pf_scoring = os.environ.get("CODA_B200_PREFILTER_SCORING", "auto")
        if self.pf_scoring not in PREFILTER_SCORING:
            raise ValueError(f"CODA_B200_PREFILTER_SCORING must be one of {PREFILTER_SCORING}, got {self.pf_scoring!r}")
        if self.pf_scoring == "sample" and self.pf_m and mode != "incremental":
            raise ValueError("CODA_B200_PREFILTER_SCORING=sample needs mode='incremental' (the template rows are cached)")
        self.sample_scoring, self.sw = False, None
        self.profile, self.profile_only = None, None
        self.xchg = None                                      # set by the group (dist.py) before the first exchange
        self._mailbox = None
        self._pi_tc, self._pi_scratch = None, None           # tensor-core marginal pass: decided on first use
        self.cidx = None                                      # compact slab: inverted index (see _build_compact_index)
        self.stream = torch.cuda.Stream(device=self.dev) if own_stream else None
        self.side = torch.cuda.Stream(device=self.dev)
        self.ev_fork, self.ev_join, self.ev_tables = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()
        self.graphs = {}
        self.loop_launches = {}                               # graph key -> launches of one replay
        self.labels_ptr = None
        # a private slot of the device's constant-memory term table (several selectors / shards may share a device)
        self.const_slot = _acquire_const_slot(self.dev.index, H) if os.environ.get("CODA_B200_R1_CONST", "1") != "0" else -1
        with self._on():
            self._alloc_static()

    # ------------------------------------------------------------------------------ utils
    @contextlib.contextmanager
    def _on(self):
        """Run the body with this shard's device current and, if it owns one, its stream current."""
        with torch.cuda.device(self.dev):
            if self.stream is not None:
                with torch.cuda.stream(self.stream):
                    yield
            else:
                yield

    def _cur(self):
        return torch.cuda.current_stream(self.dev)

    def _s(self):
        return self._cur().cuda_stream

    def sync(self):
        (self.stream or torch.cuda.current_stream(self.dev)).synchronize()

    def _call(self, name, *args, n=1):
        prof = self.profile
        key = name[:-2] if name.endswith("_x") else name         # a slab entry point's 16-bit twin times under its name
        if prof is not None and (self.profile_only is None or key in self.profile_only):
            st = self._cur()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(st)
            rc = getattr(self.lib, name)(*args)
            e1.record(st)
            prof.setdefault(key, []).append((e0, e1))
        else:
            rc = getattr(self.lib, name)(*args)
        nat.check(rc, name)
        self.counters["launches"] += n

    def start_profile(self, only=None):
        """Bracket every C-ABI launch (or just ``only``) with CUDA events on the launching stream (eager steps only)."""
        self.profile, self.profile_only = {}, (set(only) if only else None)

    def stop_profile(self):
        """-> {entry point: (launches, total ms, max ms)}; synchronises."""
        torch.cuda.synchronize(self.dev)
        out = {}
        for k, v in (self.profile or {}).items():
            ts = [a.elapsed_time(b) for a, b in v]
            out[k] = (len(ts), float(sum(ts)), float(max(ts)))
        self.profile = None
        return out

    def _slab_call(self, name, *args, n=1, base=None):
        """An entry point that reads the slab (or, ``base``, a chunk of it or the host-mode shadow): the fp32 one, or
        its ``_x`` twin with the slab's element type."""
        base = _ptr(self.preds) if base is None else base
        if self.fmt == nat.SLAB_F32:
            self._call(name, base, *args, n=n)
        else:
            self._call(name + "_x", base, self.fmt, *args, n=n)

    def _z(self, shape, dtype):
        return torch.zeros(shape, dtype=dtype, device=self.dev)

    def _e(self, shape, dtype):
        return torch.empty(shape, dtype=dtype, device=self.dev)

    # --------------------------------------------------------------------------- buffers
    def _alloc_static(self):
        H, N, C, Hp, P = self.H, self.N, self.C, self.Hp, self.P
        self.hard = self._e((N, H), torch.int16)              # uint16 bit patterns
        self.pseudo = self._e((N,), torch.int32)
        self.disagree = self._e((N,), torch.uint8)
        self.labeled = self._z((N,), torch.uint8)
        # soft-confusion sums (coda.py:42), int64 fixed point; the compact slab adds one "every column" term per row
        self.conf_buf = self._z((H * C * C + H * C,), torch.int64)
        self.conf_fx = self.conf_buf[: H * C * C].view(H, C, C)
        self.conf_rest = self.conf_buf[H * C * C:].view(H, C) if self.compact is not None else None
        self.D = self._e((H, C, C), torch.float32)
        # 16 bytes of slack behind U: the bulk-TMA marginal refresh rounds the last tile's copy up to 16 bytes
        self.U = self._e((N * C + 4,), torch.float32)[: N * C].view(N, C)
        self.pisum = self._z((C,), torch.int64)               # THIS shard's column sums (summed over shards in step_mixture)
        self.grid = torch.linspace(1e-6, 1 - 1e-6, P).to(self.dev)   # coda.py:86, built on the host (trap T1)
        self.dL = self._e((C, H, P), torch.float32)
        self.G0T = self._z((C, P, Hp), torch.float32)
        self.G1T = self._z((C, P, Hp), torch.float32)
        self.PB = self._z((C, Hp), torch.float32)
        # bf16 limb tables in tensor-core operand order (pairs_tc.cu); SIMT kernel (pairs.cu) when Hp > 256
        self.use_tc = Hp <= 256 and os.environ.get("CODA_B200_TC", "1") != "0"
        self.dLb = self._z((C, Hp // 32, 3, 256 * 32), torch.bfloat16) if self.use_tc else None
        self.Gb = self._z((C, 16, 4, Hp * 16), torch.bfloat16) if self.use_tc else None
        self.pi_hat = self._z((C,), torch.float32)
        self.m0 = self._z((Hp,), torch.float32)
        self.hb = self._z((1,), torch.float32)
        self.best_model = self._z((1,), torch.int64)
        self.eig = self._z((N,), torch.float32)
        self.nblocks = int(self.lib.coda_b200_eig_blocks(N, H, C))
        self.partials = self._z((self.nblocks, nat.REC_WORDS), torch.int64)
        # report block: one D2H copy per API step.  [flags | record (8) | tie hdr (2) | pad | tie idx | tie val]
        self.rep = self._z((REP_WORDS,), torch.int64)
        self.flags = self.rep[0:1].view(torch.int32)[0:1]
        self.bestrec = self.rep[1:9]
        self.tie_hdr = self.rep[9:11]
        self.tie_idx = self.rep[12:12 + TIE_CAP]
        self.tie_val = self.rep[12 + TIE_CAP:].view(torch.float32)[:TIE_CAP]
        self.rep_all = self._z((self.world, REP_WORDS), torch.int64)
        self.rep_host = torch.zeros((self.world, REP_WORDS), dtype=torch.int64).pin_memory()
        self.sel = self._z((2,), torch.int64)
        # staging ring for host-chosen (idx, class) records: a slot is rewritten only after its copy has executed
        self.sel_ring = torch.zeros((8, 2), dtype=torch.int64).pin_memory()
        self.sel_events = [None] * 8
        self.sel_pos = 0
        self.jvec = self._z((H,), torch.int32)
        self.terms = self._z((2 + 8 * H + 2,), torch.int64).view(torch.int32)[: 2 + 8 * H]   # 8-byte aligned
        self.step_ctr = self._z((1,), torch.int64)
        self.host_cols = self._z((1,), torch.int64) if self.host is not None else None   # host columns staged, ever
        self.n_host, self.host_slots = 0, None
        self.hist_idx = self._z((HIST_CAP,), torch.int64)
        self.hist_q = self._z((HIST_CAP,), torch.float32)
        self.hist_tie = self._z((HIST_CAP,), torch.int32)
        # ensemble sums E[n][c] (N*C floats) feed pi_rank1's majority shortcut; CODA_B200_ENS=0 disables it
        self.ens = self._e((N, C), torch.float32) if (os.environ.get("CODA_B200_ENS", "1") != "0" or self.compact is not None) else None
        cls_per_batch = max(1, min(C, TABLE_BATCH_BYTES // max(1, self.lib.coda_b200_tables_scratch_bytes(H, 1))))
        self.table_batch = int(cls_per_batch)
        self.scratch = self._e((int(self.lib.coda_b200_tables_scratch_bytes(H, self.table_batch)),), torch.uint8)

    def _make_step_struct(self):
        st = nat.StepStruct()
        st.H, st.C, st.N, st.n_offset, st.fx_shift, st.lr = self.H, self.C, self.N, self.n_offset, self.fx_shift, self.lr
        st.hard, st.labeled, st.D, st.jvec, st.sel = _ptr(self.hard), _ptr(self.labeled), _ptr(self.D), _ptr(self.jvec), _ptr(self.sel)
        st.terms = _ptr(self.terms)
        st.slot_of_model = _ptr(self.slot_of_model)
        # gather-list offsets count slab elements from the slab; the ensemble term counts fp32 elements from the
        # ensemble base (the slab itself for fp32, see ``_ens_base``)
        st.shadow_off = ((self.shadow.data_ptr() - self._slab_ptr()) // self.esz) if self.shadow is not None else 0
        st.shadow_col_stride = self.shadow_cs
        st.model_stride = self.model_stride
        ens_base = self._ens_base()
        if self.ens_shadow is not None:                                          # class-major ensemble slot
            st.ens_off = (self.ens_shadow.data_ptr() - ens_base) // 4
            st.ens_col_stride = self.shadow_cs
        else:
            st.ens_off = ((self.ens.data_ptr() - ens_base) // 4) if self.ens is not None else 0
            st.ens_col_stride = 0
        st.have_ens = 1 if self.ens is not None else 0
        st.compact_k = self.K if self.compact is not None else 0
        st.pisum_fx, st.PB, st.pi_hat, st.m0 = _ptr(self.pisum), _ptr(self.PB), _ptr(self.pi_hat), _ptr(self.m0)
        st.h_before, st.best_model = _ptr(self.hb), _ptr(self.best_model)
        st.partials, st.nblocks, st.eig, st.bestrec = _ptr(self.partials), self.nblocks, _ptr(self.eig), _ptr(self.bestrec)
        st.labels_global = None
        st.hist_idx, st.hist_q, st.hist_tie, st.hist_cap = _ptr(self.hist_idx), _ptr(self.hist_q), _ptr(self.hist_tie), HIST_CAP
        st.step_ctr = _ptr(self.step_ctr)
        st.flags = _ptr(self.flags)
        if self.host is not None and self.n_host:
            st.n_host, st.host_shadow, st.stage = self.n_host, _ptr(self.host_slots), _ptr(self.stage)
            st.stage_off = (self.stage.data_ptr() - self._slab_ptr()) // self.esz
        self.st = st

    def _slab_ptr(self):
        """Base address of the gather list's slab terms: the slab, or with a host-resident slab the device shadow
        buffer (model slots, fp32 ensemble slot, staging columns)."""
        if self.host is not None:
            return self.dshadow.data_ptr()
        return self.preds.data_ptr() if self.compact is None else 0

    def _ens_base(self):
        """fp32 base address of the ensemble term of the gather list: the slab for an fp32 slab (one base for every
        term, as the fp32 entry point reads it), the ensemble sums themselves for a 16-bit slab."""
        if self.fmt == nat.SLAB_F32 or self.ens is None:
            return self._slab_ptr()
        return self.ens_shadow.data_ptr() if self.ens_shadow is not None else self.ens.data_ptr()

    def _x(self):
        return self.xchg if (self.xchg is not None and self.world > 1) else None

    # ---------------------------------------------------------------------- construction
    # phases: scan -> [group: sum conf_fx over shards] -> posterior -> mixture (exchange) -> finish (host sync)
    def construct_scan(self):
        with self._on():
            H, N, C, s = self.H, self.N, self.C, self._s()
            if self.compact is not None:
                cs = self.compact
                self._call("coda_b200_scan_compact", _ptr(cs.ids), _ptr(cs.probs), self.model_stride, H, N, C, self.K,
                           _ptr(self.hard), _ptr(self.pseudo), _ptr(self.disagree), _ptr(self.ens), _ptr(self.flags), s)
                self._call("coda_b200_confusion_compact", _ptr(cs.ids), _ptr(cs.probs), self.model_stride,
                           _ptr(self.pseudo), H, N, C, self.K, self.fx_shift, _ptr(self.conf_fx), _ptr(self.conf_rest), s)
                self._build_compact_index()
                return
            self._record_kernels()
            # a host slab in chunks: the confusion sums are order-free integers
            walk(self.preds, lambda n0, n1, v: self._scan_range(_ptr(v), model_stride(v), n0, n1 - n0))

    def _scan_range(self, base, model_stride, n0, n):
        """The slab scan and the confusion sums of items [n0, n0 + n), read from ``base`` (their first item)."""
        H, C, s = self.H, self.C, self._s()
        pseudo = _ptr(self.pseudo[n0:])
        self._slab_call("coda_b200_scan_slab", model_stride, H, n, C, _ptr(self.hard[n0:]), pseudo,
                        _ptr(self.disagree[n0:]), _ptr(self.ens[n0:]) if self.ens is not None else None,
                        _ptr(self.flags), s, base=base)
        if self.kernels["confusion"] == "sorted":
            order = torch.argsort(self.pseudo[n0:n0 + n]).to(torch.int32)   # init-time plumbing: any grouping by label will do
            self._slab_call("coda_b200_confusion_sorted", model_stride, pseudo, _ptr(order), H, n, C, self.fx_shift,
                            _ptr(self.conf_fx), s, base=base)
            del order
        else:
            self._slab_call("coda_b200_confusion_accum", model_stride, pseudo, H, n, C, self.fx_shift,
                            _ptr(self.conf_fx), s, base=base)

    def _record_kernels(self):
        """Which construction kernels this dense slab takes, decided from the whole task (H, N, C, dtype, model
        stride): a host-resident slab, streamed in chunks, takes the kernels the same slab takes on the device.
        ``scan``: the bulk-TMA scan or the generic one (the rule of csrc/slab.cu scan_slab; chunks are whole multiples
        of its 32-item tile, so each chunk meets it exactly when the whole slab does); ``pi_full``: the tensor-core
        marginal pass or the SIMT one; ``confusion``: the pseudo-label-sorted sums or the accumulating ones."""
        H, N, C, esz = self.H, self.N, self.C, self.esz
        e16 = 16 // esz
        aligned = self.host is not None or self.preds.data_ptr() % 16 == 0
        tma = (C <= 128 and self.model_stride % e16 == 0 and (32 * C) % e16 == 0 and ((N % 32) * C) % e16 == 0
               and aligned)
        self.kernels["scan"] = "tma" if tma else "generic"
        self.kernels["confusion"] = "sorted" if C <= 128 else "accum"

    def construct_posterior(self):
        with self._on():
            H, C, s = self.H, self.C, self._s()
            self._call("coda_b200_init_dirichlets", _ptr(self.conf_fx), _ptr(self.conf_rest), H, C, self.fx_shift,
                       self.prior_strength, self.multiplier, int(self.uniform_prior), _ptr(self.D), s)
            self.conf_fx = self.conf_rest = self.conf_buf = None    # H*C*C int64, only needed once
            self._marginals_full()
            self._build_rows()

    def construct_tables(self, left: int = 1, total: int = 1):
        """Shadow slab, step struct and class tables.  Runs after every shard of the device has its row cache;
        ``left`` / ``total``: shards on this device that have still to build a shadow (this one included) / in all."""
        with self._on():
            self._build_shadow(left, total)
            self._make_step_struct()
            self._tables(0, self.C)
            self.cache_valid = False     # incremental mode: P(best | hypothetical) rows are cached once scored
            self.pending = False         # a side-stream refresh the next scoring pass has to join
            self.scored = False          # block records (`partials`) are current
            self.reported = False        # the report block in rep_host is (being) produced for the current state

    def construct_mixture(self):
        with self._on():
            self._mixture()

    def construct_finish(self):
        with self._on():
            self.check_flags(sync=True)

    def _build_compact_index(self):
        """Inverted index of the compact slab (csrc/compact.cu): per (model, class) the items whose top-K list holds the
        class.  With it the rank-1 marginal refresh reads H short lists (N K / C entries each) instead of the whole slab
        every step.  Same bytes as the slab (8 per entry): skipped when they do not fit (``CODA_B200_COMPACT_INDEX=0``
        forces the slab scan)."""
        self.cidx = None
        if os.environ.get("CODA_B200_COMPACT_INDEX", "1") == "0":
            return
        H, N, C, K, s = self.H, self.N, self.C, self.K, self._s()
        need = 8 * H * N * K + 16 * (H * C + 1) + 12 * N
        free, _total = torch.cuda.mem_get_info(self.dev)
        # leave room for what construction allocates after this point: U, the row cache (bounded by 4 * N * C * Hp bytes
        # only in the worst case; a quarter of free memory is kept back instead)
        if need > 0.5 * free:
            return
        cs = self.compact
        counts = self._z((H * C,), torch.int64)
        self._call("coda_b200_compact_index_count", _ptr(cs.ids), self.model_stride, H, N, C, K, _ptr(counts), s)
        off = self._z((H * C + 1,), torch.int64)
        torch.cumsum(counts, 0, out=off[1:])                          # construction-time plumbing
        cursor = off[:-1].clone()
        ent = self._e((H * N * K,), torch.int64)                      # {item u32, float bits} pairs
        rest = self._e((N,), torch.float32)
        self._call("coda_b200_compact_index_fill", _ptr(cs.ids), _ptr(cs.probs), self.model_stride, H, N, C, K,
                   _ptr(cursor), _ptr(ent), _ptr(rest), s, n=2)
        del counts, cursor
        self.cidx = dict(off=off, ent=ent, rest=rest, delta=self._z((N,), torch.int64))

    def _marginals_full(self):
        """coda.py:226-233 as one streaming pass; leaves THIS shard's column sums in ``pisum``."""
        H, N, C, s = self.H, self.N, self.C, self._s()
        if self.compact is not None:
            cs = self.compact
            dt = self._e((H, C, C), torch.float32)                  # D transposed + row sums: construction-time scratch
            rs = self._e((H, C), torch.float32)
            self._call("coda_b200_pi_full_compact", _ptr(cs.ids), _ptr(cs.probs), self.model_stride, _ptr(self.D), H, N, C,
                       self.K, _ptr(dt), _ptr(rs), _ptr(self.U), s, n=3)
            del dt, rs
        else:
            walk(self.preds, lambda n0, n1, v: self._pi_full(_ptr(v), model_stride(v), n0, n1 - n0))
        self._call("coda_b200_pi_reduce", _ptr(self.U), N, C, self.fx_shift, None, _ptr(self.pisum),
                   _ptr(self.flags), s)

    def _pi_full(self, base=None, model_stride=None, n0=0, n=None):
        """coda.py:227-229 over the dense slab (or items [n0, n0 + n) of it at ``base``): the wgmma kernel when the
        shape of the whole slab allows it (pi_tc.cu), else fp32 SIMT.  ``CODA_B200_PI_FULL=simt`` forces the SIMT
        kernel."""
        H, N, C, s = self.H, self.N, self.C, self._s()
        if self._pi_tc is None:
            want = os.environ.get("CODA_B200_PI_FULL", "tc") != "simt"
            if self.fmt == nat.SLAB_F32:
                aligned = self.host is not None or self.preds.data_ptr() % 16 == 0
                self._pi_tc = bool(want and self.lib.coda_b200_pi_full_tc_ok(H, N, C, self.model_stride) and aligned)
            else:
                # the tensor-core and SIMT passes differ in the last bits: a 16-bit slab takes the pass its fp32
                # widening (contiguous, aligned) would take, or stops
                tc32 = bool(self.lib.coda_b200_pi_full_tc_ok(H, N, C, N * C))
                ok = bool(self.lib.coda_b200_pi_full_tc_ok_x(self.fmt, H, N, C, self.model_stride))
                if want and tc32 and not ok:
                    raise NotImplementedError(f"coda_b200: the tensor-core marginal pass cannot read this "
                                              f"{self.preds.dtype} slab (C={C}); its fp32 widening would take it")
                self._pi_tc = bool(want and tc32)
            if self._pi_tc:
                self._pi_scratch = self._e((int(self.lib.coda_b200_pi_full_tc_scratch_bytes(H, C)),), torch.uint8)
            self.kernels["pi_full"] = "tc" if self._pi_tc else "simt"
        ms = self.model_stride if model_stride is None else model_stride
        n = N if n is None else n
        U = _ptr(self.U[n0:])
        if self._pi_tc:
            self._slab_call("coda_b200_pi_full_tc", ms, _ptr(self.D), H, n, C, U, _ptr(self._pi_scratch),
                            _ptr(self.flags), s, n=2, base=base)
        else:
            self._slab_call("coda_b200_pi_full", ms, _ptr(self.D), H, n, C, U, s, base=base)

    def _build_rows(self):
        H, N, C, W, T, s = self.H, self.N, self.C, self.W, self.T, self._s()
        ent_cnt = self._e((N,), torch.int32)
        heavy_cnt = self._e((N,), torch.int32)
        cls_heavy = self._z((C,), torch.int32)
        self._call("coda_b200_pair_count", _ptr(self.hard), H, N, C, _ptr(ent_cnt), _ptr(heavy_cnt), _ptr(cls_heavy), s)
        heavy = cls_heavy.cpu().numpy().astype(np.int64)        # host sync (construction only)
        n_ent = int(ent_cnt.sum(dtype=torch.int64).item())
        self.n_heavy = int(heavy.sum())
        self.n_entries = n_ent
        self.max_entries = int(ent_cnt.max().item())
        per_cls = 1 + H + heavy
        cls_base = np.zeros(C + 1, dtype=np.int64)
        np.cumsum(per_cls, out=cls_base[1:])
        self.npairs = int(cls_base[-1])                         # == T + n_heavy
        if self.npairs >= 2 ** 31 or n_ent >= 2 ** 31:
            raise NotImplementedError("coda_b200: more than 2^31 rows in one shard")
        self.ent_off = self._z((N + 1,), torch.int32)
        self.heavy_off = self._z((N + 1,), torch.int32)
        torch.cumsum(ent_cnt, 0, out=self.ent_off[1:])          # init-time plumbing
        torch.cumsum(heavy_cnt, 0, out=self.heavy_off[1:])
        del ent_cnt, heavy_cnt
        self.cls_base_host = cls_base
        self.cls_base = torch.from_numpy(cls_base).to(self.dev)
        # tiles of <= 32 (SIMT) or <= 128 (wgmma) same-class work-list positions
        def make_tiles(width, per_cls=per_cls):
            nt = (per_cls + width - 1) // width
            tile_off = np.zeros(C + 1, dtype=np.int64)
            np.cumsum(nt, out=tile_off[1:])
            cls_of_tile = np.repeat(np.arange(C, dtype=np.int64), nt)
            k_in_cls = np.arange(int(tile_off[-1]), dtype=np.int64) - tile_off[cls_of_tile]
            start = cls_base[cls_of_tile] + width * k_in_cls
            cnt = np.minimum(width, per_cls[cls_of_tile] - width * k_in_cls)
            tiles = np.stack([cls_of_tile, start, cnt, np.zeros_like(cnt)], axis=1).astype(np.int32)
            return tile_off, int(nt.max()), torch.from_numpy(tiles).to(self.dev)
        width = 128 if self.use_tc else 32

        def set_tiles(tiles):
            tile_off, self.max_cls_tiles, self.tiles = tiles
            self.tile_off_host = tile_off
            self.tile_off = torch.from_numpy(tile_off).to(self.dev)
            self.ntiles = int(tile_off[-1])
        set_tiles(make_tiles(width))
        self.ent_row = self._e((max(1, n_ent),), torch.int32)
        self.ent_cls = self._e((max(1, n_ent),), torch.int16)
        self.zmask = self._e((self.npairs, W), torch.int32)
        self.row_of = self._e((self.npairs,), torch.int32)
        self.row_cls = self._e((max(1, self.n_heavy),), torch.int16)
        cursor = self._z((C,), torch.int32)
        self._call("coda_b200_pair_fill", _ptr(self.hard), H, N, C, _ptr(self.ent_off), _ptr(self.heavy_off),
                   _ptr(self.cls_base), _ptr(cursor), _ptr(self.ent_row), _ptr(self.ent_cls), _ptr(self.zmask),
                   _ptr(self.row_of), _ptr(self.row_cls), s, n=2)
        # ELL copy of the entry lists when the longest one fits four entries per lane of an 8-lane group
        self.ell_row, self.ell_cls, self.ell_k = None, None, 0
        if 0 < self.max_entries <= 32 and C <= 128:
            self.ell_k = (self.max_entries + 3) // 4 * 4
            self.ell_row = self._e((N, self.ell_k), torch.int32)
            self.ell_cls = self._e((N, self.ell_k), torch.int16)
            self._call("coda_b200_ell_build", _ptr(self.ent_off), _ptr(self.ent_row), _ptr(self.ent_cls), N, self.ell_k,
                       _ptr(self.ell_row), _ptr(self.ell_cls), s)
        # sample scoring caches the T template rows only; the sample's heavy rows go to a scratch of `cap` rows
        sample = self._choose_sample_scoring()
        cap = self._sample_capacity() if sample else 0
        self.gain = None if sample else self._z((self.npairs,), torch.float32)   # every row's gain (templates first)
        self.ph_cache = None
        if self.mode == "incremental":
            need = (self.T * self.Hp * 4 + self._sample_bytes(cap)) if sample else self.npairs * self.Hp * 4
            free, _total = torch.cuda.mem_get_info(self.dev)
            if need + (2 << 30) > free + torch.cuda.memory_reserved(self.dev) - torch.cuda.memory_allocated(self.dev):
                # the row cache does not fit next to the slab: fall back to recomputing the rows every step
                import warnings
                warnings.warn(f"coda_b200: row cache of {need / 2 ** 30:.1f} GiB does not fit "
                              f"({free / 2 ** 30:.1f} GiB free); falling back to mode='recompute'")
                self.mode = "recompute"
                if sample:
                    self.gain = self._z((self.npairs,), torch.float32)
                sample = False
            else:
                self.ph_cache = self._e((self.T if sample else self.npairs, self.Hp), torch.float32)
        self.sample_scoring = sample
        if sample:
            # the tile lists cover the template positions only: the cache fill and the class-t refresh touch no
            # heavy row (row ids < T, so they land in the T cached rows)
            set_tiles(make_tiles(width, np.full(C, 1 + H, dtype=np.int64)))
            self._alloc_sample(cap)

    def _choose_sample_scoring(self) -> bool:
        """prefilter_n = m: score only the m sampled items (sample.cu) instead of every item.  Chosen when the
        sample's heavy rows cost less to integrate than all cached rows cost to stream (m * R <= N), in incremental
        mode only: the sampled scoring reads the cached template rows.  CODA_B200_PREFILTER_SCORING forces a side."""
        if self.pf_m <= 0 or self.pf_scoring == "full" or self.mode != "incremental":
            return False
        return self.pf_scoring == "sample" or self.pf_m * PREFILTER_ROW_COST_RATIO <= self.n_global

    def _sample_capacity(self) -> int:
        """Heavy rows of the m items that have the most: the most one sample (or one chunk of m items) can hold."""
        heavy = self.heavy_off[1:] - self.heavy_off[:-1]
        return max(1, int(torch.topk(heavy, min(self.pf_m, self.N)).values.sum()) if self.n_heavy else 0)

    def _sample_bytes(self, cap) -> int:
        """Device bytes of the sampled pass's scratch (see _alloc_sample)."""
        width = 128 if self.use_tc else 32
        m, C = self.pf_m, self.C
        return cap * (self.Hp * 4 + self.W * 4 + 4 + 2 + 4) + self.T * 4 + (cap // width + C + 1) * 16 + 8 * m + 4 * C

    def _alloc_sample(self, cap):
        """Scratch of the sampled scoring pass, sized for the m items with the most heavy rows."""
        H, C, W, Hp, T, m = self.H, self.C, self.W, self.Hp, self.T, self.pf_m
        width = 128 if self.use_tc else 32
        maxtiles = cap // width + C + 1
        self.sw = dict(cap=cap, width=width, maxtiles=maxtiles,
                       items=self._z((m,), torch.int32), hoff=self._z((m + 1,), torch.int32),
                       cursor=self._z((C,), torch.int32), tiles=self._z((maxtiles, 4), torch.int32),
                       tile_off=self._z((2,), torch.int64), sel=self._z((2,), torch.int64),
                       nheavy=self._z((1,), torch.int64), zmask=self._z((cap, W), torch.int32),
                       row_of=self._z((cap,), torch.int32), row_cls=self._z((cap,), torch.int16),
                       rows=self._e((cap, Hp), torch.float32), gain=self._z((T + cap,), torch.float32),
                       all_items=None)

    def shadow_reserve(self) -> int:
        """Device bytes this shard leaves free when it sizes its shadow: what it still allocates after construction
        (the largest is a U-sized ``pi_hat_xi`` read-out; graph instantiation, lazily loaded kernels, the report and
        history read-outs are small) plus a 1 GiB margin for the caller.  ``CODA_B200_SHADOW_RESERVE_GB`` overrides."""
        env = os.environ.get("CODA_B200_SHADOW_RESERVE_GB")
        base = int(float(env) * 2 ** 30) if env is not None else 4 * self.N * self.C + (1 << 30)
        if self.host is not None:
            # a host-resident slab also keeps, at worst, two staging columns per model, and the shadow pass streams the
            # slab through two chunk buffers (plus one widening chunk)
            from .datasets import DEFAULT_CHUNK_BYTES
            base += 2 * self.H * self._shadow_cs() * self.esz + 2 * self.host.chunk_bytes() + DEFAULT_CHUNK_BYTES
        return base

    def _shadow_cs(self):
        """Column stride of the shadow: every (slot, class) column starts 16-byte aligned."""
        return (self.N + 7) // 8 * 8 if self.esz == 2 else (self.N + 3) // 4 * 4

    def _build_shadow(self, left: int = 1, total: int = 1):
        """Class-major shadow copy of the ensemble sums and of as many models as spare HBM allows (least accurate
        first): slots [0, n_shadow) hold models, slot n_shadow (when present) holds E.  ``left`` / ``total``: shards on
        this device that have still to build a shadow (this one included) / in all -- each takes an equal share of
        what is free once every shard's reserve is set aside."""
        self.shadow, self.slot_of_model, self.n_shadow, self.shadow_cs = None, None, 0, 0
        self.ens_shadow = None
        host = self.host is not None
        if not host and (self.mode == "recompute_all" or os.environ.get("CODA_B200_SHADOW", "1") == "0"
                         or self.compact is not None):
            return
        H, N, C = self.H, self.N, self.C
        cs = self._shadow_cs()
        cap = os.environ.get("CODA_B200_SHADOW_MODELS")
        want = H if cap is None else max(0, min(H, int(cap)))
        order = None
        if want > 0 or host:
            # disagreement of every model with the ensemble pseudo-label: the models that will need gathers most often
            dis = torch.zeros(H, dtype=torch.int64, device=self.dev)
            step = max(1, (64 << 20) // max(1, H))
            for n0 in range(0, N, step):
                blk = self.hard[n0:n0 + step].to(torch.int32) & 0xFFFF
                dis += (blk != self.pseudo[n0:n0 + step, None]).sum(0)
            order = torch.argsort(dis, descending=True, stable=True).to(torch.int32)
            del dis, blk
        torch.cuda.synchronize(self.dev)
        torch.cuda.empty_cache()                                # the temporaries above are not spare memory
        free, _total = torch.cuda.mem_get_info(self.dev)
        # model slots hold the slab's own element type (exact); the ensemble slot is fp32
        S, ne = shadow_slots(free, self.shadow_reserve(), cs * C * self.esz, want, self.ens is not None, left, total,
                             ens_slot_bytes=cs * C * 4)
        if host:
            self._build_host_shadow(order, S, ne, cs)
            return
        if S + ne == 0:
            return
        slot = torch.full((H,), -1, dtype=torch.int32, device=self.dev)
        if self.esz == 4:
            self.shadow = self._e((S + ne, C, cs), torch.float32)
            self.ens_shadow = self.shadow[S] if ne else None
        else:                                                   # a 16-bit slab: E in a buffer of its own
            self.shadow = self._e((S, C, cs), self.preds.dtype) if S > 0 else None
            self.ens_shadow = self._e((C, cs), torch.float32) if ne else None
        if S > 0:
            order = order[:S].contiguous()
            slot[order.long()] = torch.arange(S, dtype=torch.int32, device=self.dev)
            self._slab_call("coda_b200_shadow_build", self.model_stride, H, N, C, _ptr(order), S, cs,
                            _ptr(self.shadow), self._s())
        if ne:                                                  # E [N][C] is a one-model slab
            first = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self._call("coda_b200_shadow_build", _ptr(self.ens), N * C, 1, N, C, _ptr(first), 1, cs,
                       _ptr(self.ens_shadow), self._s())
        self.slot_of_model, self.n_shadow, self.shadow_cs = slot, S, cs

    def _build_host_shadow(self, order, S, ne, cs):
        """A host-resident slab: every model gets a shadow slot.  ``order`` (least accurate first) puts models
        [0, S) in device slots and the rest in pinned host slots [H - S][C][cs] at the slab's width, mapped for the
        device; both are transposed from each chunk as the slab streams through.  One device buffer ``dshadow`` holds
        the device slots, the fp32 ensemble slot (fp32 slab) and the 2 (H - S) staging columns of k_host_stage: it is
        the base every slab term of the gather list counts from."""
        H, N, C, esz, s = self.H, self.N, self.C, self.esz, self._s()
        nh = H - S
        ne_in = ne if esz == 4 else 0                           # the fp32 ensemble slot shares the buffer
        self.dshadow = self._e(((S + ne_in) * C * cs + max(1, 2 * nh) * cs,), self.host.dtype)
        if S + ne_in:
            self.shadow = self.dshadow[: (S + ne_in) * C * cs].view(S + ne_in, C, cs)
        if ne:
            self.ens_shadow = self.shadow[S] if ne_in else self._e((C, cs), torch.float32)
        self.stage = self.dshadow[(S + ne_in) * C * cs:]
        self.host_slots = _PinnedHost((nh, C, cs), self.host.dtype, self.lib) if nh else None
        self.n_host = nh
        slot = torch.empty((H,), dtype=torch.int32, device=self.dev)
        slot[order.long()] = torch.arange(H, dtype=torch.int32, device=self.dev)
        dev_order, host_order = order[:S].contiguous(), order[S:].contiguous()

        def body(n0, n1, v):
            n = n1 - n0
            if S:
                self._slab_call("coda_b200_shadow_build", n * C, H, n, C, _ptr(dev_order), S, cs,
                                _ptr(self.shadow) + n0 * esz, s, base=_ptr(v))
            if nh:                                              # written straight into the mapped host slots
                self._slab_call("coda_b200_shadow_build", n * C, H, n, C, _ptr(host_order), nh, cs,
                                _ptr(self.host_slots) + n0 * esz, s, base=_ptr(v))
        self.host.walk(body)
        if ne:
            first = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self._call("coda_b200_shadow_build", _ptr(self.ens), N * C, 1, N, C, _ptr(first), 1, cs,
                       _ptr(self.ens_shadow), s)
        self.slot_of_model, self.n_shadow, self.shadow_cs = slot, S, cs

    # ------------------------------------------------------------------------ step pieces (enqueue only)
    def _tables(self, lo, hi, sel=False):
        H, C, s = self.H, self.C, self._s()
        if sel:
            self._call("coda_b200_beta_tables", _ptr(self.D), _ptr(self.grid), H, C, self.P, self.hyp_w, 0, 1,
                       _ptr(self.sel), _ptr(self.scratch), _ptr(self.dL), _ptr(self.G0T), _ptr(self.G1T),
                       _ptr(self.PB), _ptr(self.dLb), _ptr(self.Gb), _ptr(self.flags), s, n=3)
            return
        for b0 in range(lo, hi, self.table_batch):
            b1 = min(hi, b0 + self.table_batch)
            self._call("coda_b200_beta_tables", _ptr(self.D), _ptr(self.grid), H, C, self.P, self.hyp_w, b0, b1, None,
                       _ptr(self.scratch), _ptr(self.dL), _ptr(self.G0T), _ptr(self.G1T), _ptr(self.PB),
                       _ptr(self.dLb), _ptr(self.Gb), _ptr(self.flags), s, n=3)

    def _mixture(self):
        self._call("coda_b200_step_mixture", self.st, self._x(), self._s())

    def _pair_rows(self, tile_lo, tile_hi, gains=True, sel=False):
        tail = (_ptr(self.PB), _ptr(self.m0) if gains else None, _ptr(self.pi_hat) if gains else None, self.H,
                _ptr(self.ph_cache), _ptr(self.gain) if gains else None, _ptr(self.sel) if sel else None,
                _ptr(self.tile_off) if sel else None, _ptr(self.flags), self._s())
        if self.use_tc:
            self._call("coda_b200_pair_rows_tc", _ptr(self.tiles), int(tile_lo), int(tile_hi), _ptr(self.zmask),
                       _ptr(self.row_of), _ptr(self.dLb), _ptr(self.Gb), *tail)
        else:
            self._call("coda_b200_pair_rows", _ptr(self.tiles), int(tile_lo), int(tile_hi), _ptr(self.zmask),
                       _ptr(self.row_of), _ptr(self.dL), _ptr(self.G0T), _ptr(self.G1T), *tail)

    def _score(self):
        """coda.py:235-281 + the per-block arg-max of coda.py:306/309 -> ``partials``."""
        if self.scored:
            return
        if self.sample_scoring:
            raise RuntimeError("coda_b200: this engine scores only prefilter samples (no heavy-row cache); the full "
                               "scoring pass is not available (CODA_B200_PREFILTER_SCORING=full keeps it)")
        if self.mode == "incremental":
            if not self.cache_valid:
                self._pair_rows(0, self.ntiles, gains=False)    # fill the row cache once
                self.cache_valid = True
            if self.pending:
                self._cur().wait_event(self.ev_join)            # the class-t rows of the side stream
                self.pending = False
            # template rows + heavy rows in one stream
            self._call("coda_b200_row_gains", _ptr(self.ph_cache), _ptr(self.row_cls), self.n_heavy, self.H, self.C,
                       _ptr(self.PB), _ptr(self.m0), _ptr(self.pi_hat), _ptr(self.gain), self._s())
        else:
            if self.pending:
                self._cur().wait_event(self.ev_join)
                self.pending = False
            self._pair_rows(0, self.ntiles)
        self._call("coda_b200_gain_eig", _ptr(self.U), self.N, self.C, self.H, _ptr(self.ent_off), _ptr(self.ent_row),
                   _ptr(self.ent_cls), _ptr(self.gain), _ptr(self.labeled), _ptr(self.disagree), self.n_offset,
                   self.max_entries, _ptr(self.ell_row), _ptr(self.ell_cls), self.ell_k, _ptr(self.eig),
                   _ptr(self.partials), _ptr(self.flags), self._s())
        self.scored = True

    def _score_sample(self):
        """eig of the items in ``sw['items']`` only (sample.cu): their heavy rows as a work list, integrated into the
        scratch by the row kernel in its device-``sel`` form, the gains of the template rows and the scratch, then the
        assembly.  Every other entry of ``eig`` keeps its value."""
        H, C, s, sw, m = self.H, self.C, self._s(), self.sw, self.pf_m
        if not self.cache_valid:
            self._pair_rows(0, self.ntiles, gains=False)    # the template rows (the cache is filled once)
            self.cache_valid = True
        common = (_ptr(self.ent_off), _ptr(self.ent_row), _ptr(self.ent_cls), _ptr(self.heavy_off))
        self._call("coda_b200_sample_plan", _ptr(sw["items"]), m, *common, H, C, sw["width"], _ptr(sw["hoff"]),
                   _ptr(sw["cursor"]), _ptr(sw["tiles"]), _ptr(sw["tile_off"]), _ptr(sw["nheavy"]), s)
        self._call("coda_b200_sample_fill", _ptr(sw["items"]), m, _ptr(self.hard), H, C, *common, _ptr(sw["hoff"]),
                   _ptr(sw["cursor"]), _ptr(sw["zmask"]), _ptr(sw["row_of"]), _ptr(sw["row_cls"]), s)
        tail = (_ptr(self.PB), None, None, H, _ptr(sw["rows"]), None, _ptr(sw["sel"]), _ptr(sw["tile_off"]),
                _ptr(self.flags), s)
        if self.use_tc:
            self._call("coda_b200_pair_rows_tc", _ptr(sw["tiles"]), 0, sw["maxtiles"], _ptr(sw["zmask"]),
                       _ptr(sw["row_of"]), _ptr(self.dLb), _ptr(self.Gb), *tail)
        else:
            self._call("coda_b200_pair_rows", _ptr(sw["tiles"]), 0, sw["maxtiles"], _ptr(sw["zmask"]),
                       _ptr(sw["row_of"]), _ptr(self.dL), _ptr(self.G0T), _ptr(self.G1T), *tail)
        if self.pending:
            self._cur().wait_event(self.ev_join)            # the class-t template rows of the side stream
            self.pending = False
        self._call("coda_b200_sample_gains", _ptr(self.ph_cache), _ptr(sw["rows"]), _ptr(sw["row_cls"]), sw["cap"],
                   _ptr(sw["nheavy"]), H, C, _ptr(self.PB), _ptr(self.m0), _ptr(self.pi_hat), _ptr(sw["gain"]), s)
        self._call("coda_b200_sample_eig", _ptr(sw["items"]), m, _ptr(sw["hoff"]), _ptr(self.U), C, H, *common,
                   _ptr(sw["gain"]), self.max_entries, _ptr(self.eig), _ptr(self.flags), s)

    def score_items(self, local_ids):
        """Sample scoring: eig of the local items ``local_ids`` (a CPU or device integer tensor; None = every item of
        the shard), in chunks of the scratch capacity (prefilter_n items).  One upload, then device copies; enqueue
        only."""
        m, items = self.pf_m, self.sw["items"]
        with self._on():
            if local_ids is None:
                if self.sw["all_items"] is None:
                    self.sw["all_items"] = torch.arange(self.N, dtype=torch.int32, device=self.dev)
                ids = self.sw["all_items"]
            elif local_ids.device == self.dev:
                ids = local_ids.to(torch.int32)
            else:
                ids = local_ids.to(torch.int32).pin_memory().to(self.dev, non_blocking=True)
            for c0 in range(0, ids.numel(), m):
                chunk = ids[c0:c0 + m]
                if chunk.numel() < m:
                    items.fill_(-1)
                items[: chunk.numel()].copy_(chunk)
                self._score_sample()

    def pf_fallback_score(self):
        """run_steps, all-unlabeled fallback with more candidates than the sample holds (coda.py:239: every unlabeled
        item is scored): eig of every item in chunks, then the block records of the EIG pass from it."""
        with self._on():
            self.score_items(None)
            self._call("coda_b200_static_records", _ptr(self.eig), _ptr(self.labeled), _ptr(self.disagree), self.N,
                       self.n_offset, self.nblocks, _ptr(self.partials), self._s())

    def pf_fallback_commit(self, rule, record_best):
        """The EIG loop's selection over those records (its tie rule), the label and the posterior update."""
        with self._on():
            self._select(self.eig, rule)
            self._post_label()
            if record_best:
                self._record_best()

    def _post_label(self):
        """coda.py:317-319 after ``sel`` / ``jvec`` / D / the gather list are in place (step_select or step_label):
        marginal refresh + the tables that depend on the new D.  incremental / recompute: the class-t tables (and the
        cached rows of the class-t work list) only need the new D, so they are rebuilt on a side stream while the main
        stream does the HBM-bound marginal refresh; the mixture waits for the tables, the next scoring pass for the rows."""
        H, N, C, s = self.H, self.N, self.C, self._s()
        self.scored = False
        self.reported = False
        if self.mode == "recompute_all":
            self._pi_full()
            self._call("coda_b200_pi_reduce", _ptr(self.U), N, C, self.fx_shift, None, _ptr(self.pisum), _ptr(self.flags), s)
            self._tables(0, C)
            self._mixture()
            return
        main = self._cur()
        refresh_rows = self.mode == "incremental" and self.cache_valid
        fork = self.overlap
        if fork:
            self.ev_fork.record(main)
            self.side.wait_event(self.ev_fork)
            ctx = torch.cuda.stream(self.side)
        else:
            ctx = contextlib.nullcontext()
        with ctx:
            self._tables(0, 1, sel=True)
            if fork:
                self.ev_tables.record(self.side)
            if refresh_rows:     # cached rows of the class-t work list (no gains: m0 / pi_hat are not final yet)
                self._pair_rows(0, self.max_cls_tiles, gains=False, sel=True)
            if fork:
                self.ev_join.record(self.side)
        if self.compact is not None and self.cidx is not None:
            ix = self.cidx
            self._call("coda_b200_pi_rank1_index", _ptr(ix["off"]), _ptr(ix["ent"]), _ptr(ix["rest"]), _ptr(self.jvec), H, N, C,
                       _ptr(self.sel), self.lr, self.fx_shift, _ptr(self.terms), _ptr(ix["delta"]), _ptr(self.U),
                       _ptr(self.pisum), _ptr(self.flags), s, n=2)
        elif self.compact is not None:
            cs = self.compact
            self._call("coda_b200_pi_rank1_compact", _ptr(cs.ids), _ptr(cs.probs), self.model_stride, _ptr(self.ens), H, N,
                       C, self.K, _ptr(self.sel), self.lr, self.fx_shift, _ptr(self.terms), _ptr(self.U),
                       _ptr(self.pisum), _ptr(self.flags), s)
        else:
            base = None
            if self.host is not None:                           # host-slot columns -> staging columns, terms rewritten
                self._call("coda_b200_host_stage", self.st, self.fmt, _ptr(self.host_cols), s, n=2)
                base = self._slab_ptr()
            ens = _ptr(self.ens) if self.fmt == nat.SLAB_F32 else self._ens_base()
            self._slab_call("coda_b200_pi_rank1", ens, H, N, C, _ptr(self.sel), self.lr,
                            self.fx_shift, _ptr(self.terms), _ptr(self.U), _ptr(self.pisum), _ptr(self.flags),
                            4 if fork else 8, self.const_slot, s, base=base)
        if fork:
            main.wait_event(self.ev_tables)     # the mixture needs PB[t]; the rows are awaited by the scoring pass
            self.pending = True
        self._mixture()

    # ------------------------------------------------------------------------ host-free loop
    # One step body for every acquisition of CODA.run_steps, captured as one CUDA graph per (kind, record_best, rule):
    #   "eig"           step_select over the scoring pass's block records -> refresh + mixture -> the scoring pass for
    #                   the next step
    #   "uncertainty"   block records from the static scores -> step_select -> refresh + mixture (no scoring pass)
    #   "iid"           candidate ties -> k-th of them (pre-drawn k) -> commit -> step_label -> refresh + mixture
    #   "prefilter"     candidate ties -> sampled positions resolved and reduced -> commit -> step_label -> refresh +
    #                   mixture, then the scoring pass for the next step (with sample scoring a step scores its sample)
    #   "prefilter_id"  the prefilter with the identity sample (sample scoring, steps with at most prefilter_n candidates)
    # rule "reference" breaks isclose ties from the replica of Python's generator (ref_bind); record_best appends
    # best_model -> hist_best.  The pre-draws of iid / prefilter (one row of `width` int64 per step,
    # include/coda_b200.h) are replayed from a device buffer of `rows` rows that the caller refills chunk by chunk
    # (abl_load).
    def _bind_labels(self, labels_dev):
        if labels_dev.data_ptr() != self.labels_ptr:
            if labels_dev.dtype != torch.int64 or labels_dev.device != self.dev or labels_dev.numel() < self.n_global:
                raise ValueError("labels_dev must be an int64 tensor of all n_global labels on this shard's device")
            self.st.labels_global = labels_dev.data_ptr()
            self.labels_ptr = labels_dev.data_ptr()
            self._labels_keep = labels_dev
            for key in [k for k in self.graphs if isinstance(k, tuple) and k[0] == "loop"]:
                del self.graphs[key]

    def _loop_body(self, kind="eig", record_best=False, rule="first"):
        """One step: the kind's selection, the posterior update, the scoring pass for the next selection (see
        ``_loop_scores``), and with ``record_best`` the step's best model."""
        if kind == "eig":
            self._select(self.eig, rule)
        elif kind == "uncertainty":
            self._call("coda_b200_static_records", _ptr(self.abl_score), _ptr(self.labeled), _ptr(self.disagree), self.N,
                       self.n_offset, self.nblocks, _ptr(self.partials), self._s())
            self._select(self.abl_score, rule)
        else:
            self._select_drawn(kind, rule)
        self._post_label()
        if self._loop_scores(kind):
            self._score()
        if record_best:
            self._record_best()

    def _loop_scores(self, kind):
        """Whether the loop body of ``kind`` ends with the full scoring pass (the next step selects from it)."""
        return kind == "eig" or (kind == "prefilter" and not self.sample_scoring)

    def _select(self, v, rule):
        """step_select over the block records; tie_rule="reference": the deferring select, and a step it leaves
        pending draws its pick over score ``v`` from the Python generator's replica (_ref_tie)."""
        if rule == "reference":
            self._call("coda_b200_step_select_defer", self.st, self._x(), _ptr(self.ref_lw[3:]), self._s())
            self._ref_tie(v)
        else:
            self._call("coda_b200_step_select", self.st, self._x(), self._s())

    def _record_best(self):
        """best_model (written by step_mixture on this stream) -> hist_best[step_ctr - 1]."""
        self._call("coda_b200_record_best", _ptr(self.best_model), _ptr(self.step_ctr), _ptr(self.hist_best),
                   HIST_CAP, self._s())

    def _ref_tie(self, v):
        """A pending step's band of isclose candidates over score ``v`` -> _randbelow draw -> commit -> label."""
        s, x, pend = self._s(), self._x(), _ptr(self.ref_lw[3:])
        self._call("coda_b200_tie_band", _ptr(v), _ptr(self.labeled), _ptr(self.disagree), self.N, _ptr(self.bestrec),
                   pend, _ptr(self.ref_xp), s)
        self._call("coda_b200_tie_draw", self.st, _ptr(v), _ptr(self.disagree), _ptr(self.ref_xp), pend,
                   _ptr(self.pyrng), _ptr(self.ref_lw), x, s)
        self._call("coda_b200_step_label_if", self.st, x, pend, s)

    def _select_drawn(self, kind, rule):
        """iid / prefilter / prefilter_id: the candidates, the pick from this step's pre-draw row, the label.
        tie_rule="reference" (prefilter): the row is drawn on the device and ties from the same generator; iid's
        pre-drawn rows already are the reference's draws."""
        s, x, pre, w = self._s(), self._x(), self.abl_pre, self.abl_width
        ref = rule == "reference" and kind != "iid"
        lw = self.ref_lw if ref else self.abl_lw
        self._call("coda_b200_select_extreme_xchg", _ptr(self.abl_cand), _ptr(self.labeled), self.N, 1,
                   _ptr(self.abl_xp), _ptr(self.abl_best), x, _ptr(self.flags), s, n=2)
        if kind == "iid":
            self._call("coda_b200_abl_draw", _ptr(pre), w, _ptr(lw), s)
            self._call("coda_b200_select_kth_xchg_dev", _ptr(self.abl_cand), _ptr(self.labeled), self.N,
                       _ptr(self.abl_xp), _ptr(self.abl_best), _ptr(lw[1:]), _ptr(lw[2:]), self.n_offset,
                       _ptr(self.abl_pick), x, _ptr(self.flags), s)
            self._call("coda_b200_abl_commit", self.st, _ptr(self.abl_best), _ptr(self.abl_pick), _ptr(pre), w,
                       _ptr(lw), s)
        else:
            if kind == "prefilter_id":
                self._call("coda_b200_pf_identity", _ptr(self.abl_best), _ptr(pre), w - 1, _ptr(lw), _ptr(self.flags), s)
            elif ref:
                self._call("coda_b200_pf_sample", _ptr(self.abl_best), _ptr(pre), w - 1, self.ref_setsize,
                           _ptr(self.pyrng), _ptr(self.ref_pool), _ptr(self.ref_seen), _ptr(lw), _ptr(self.flags), s)
            self._pf_score_sample(pre, w, lw)
            self._call("coda_b200_prefilter_pick", _ptr(self.eig), _ptr(self.abl_cand), _ptr(self.labeled), self.N,
                       self.n_offset, _ptr(self.abl_xp), _ptr(self.abl_best), _ptr(pre), w, w - 1, _ptr(lw),
                       _ptr(self.abl_recs), s)
            if ref:
                pend = _ptr(lw[3:])
                self._call("coda_b200_prefilter_commit_defer", self.st, _ptr(self.abl_recs), self.abl_nrec,
                           _ptr(self.abl_best), _ptr(pre), w, _ptr(lw), pend, x, s)
                self._call("coda_b200_pf_band", _ptr(self.eig), _ptr(self.abl_cand), _ptr(self.labeled), self.N,
                           self.n_offset, _ptr(self.abl_xp), _ptr(self.abl_best), _ptr(pre), w, w - 1, _ptr(lw), pend,
                           _ptr(self.ref_band), s)
                self._call("coda_b200_pf_tie_draw", self.st, _ptr(self.ref_band), w - 1, pend, _ptr(self.pyrng),
                           _ptr(self.ref_bits), _ptr(lw), x, s)
            else:
                self._call("coda_b200_prefilter_commit", self.st, _ptr(self.abl_recs), self.abl_nrec,
                           _ptr(self.abl_best), _ptr(pre), w, _ptr(lw), x, s)
        self._call("coda_b200_step_label", self.st, x, s)

    def _pf_score_sample(self, pre, w, lw):
        """With sample scoring: this step's sample positions -> local items (as prefilter_pick resolves them) -> their
        eig, which prefilter_pick then reads."""
        if self.sample_scoring:
            self._call("coda_b200_pf_resolve", _ptr(self.abl_cand), _ptr(self.labeled), self.N, _ptr(self.abl_xp),
                       _ptr(self.abl_best), _ptr(pre), w, w - 1, _ptr(lw), _ptr(self.sw["items"]), self._s())
            self._score_sample()

    def device_step(self, labels_dev: torch.Tensor, step: int | None = None, hist_idx=None, hist_q=None):
        """One acquisition step with no host round trip: pick the arg-max (first index on equal values, coda.py:309;
        an isclose tie that the reference would break with random.choice is recorded in ``hist_tie``), look the label
        up on the device (coda/oracle.py:23-24), update the posterior, score the next selection.  Eager launches of the
        "eig" loop body; see the phases below for the CUDA-graph loop.  ``hist_idx`` / ``hist_q``: optional
        caller-owned history (slot = step)."""
        with self._on():
            self._bind_labels(labels_dev)
            if step is not None:
                self.step_ctr.fill_(int(step))
            self._score()
            self._loop_body()
            if hist_idx is not None and step is not None:
                hist_idx[step] = self.hist_idx[int(step) % HIST_CAP]
                if hist_q is not None:
                    hist_q[step] = self.hist_q[int(step) % HIST_CAP]

    # The graph loop in phases, so that a front end driving several shards from one thread never blocks on a shard
    # whose peers have not been enqueued yet: prepare (no exchange inside) -> one eager step -> capture -> replays.
    # The defaults are the EIG loop with the first maximum of a tie and no best-model record.
    def loop_prepare(self, labels_dev: torch.Tensor, record_best: bool = False, kind: str = "eig"):
        with self._on():
            self._bind_labels(labels_dev)
            if record_best and getattr(self, "hist_best", None) is None:
                self.hist_best = torch.full((HIST_CAP,), -1, dtype=torch.int32, device=self.dev)
            if self._loop_scores(kind):
                self._score()

    def loop_ready(self, record_best: bool = False, rule: str = "first", kind: str = "eig") -> bool:
        return (not self.use_graph) or self.graphs.get(("loop", kind, bool(record_best), rule)) is not None

    def loop_eager(self, record_best: bool = False, rule: str = "first", kind: str = "eig"):
        with self._on():
            self._loop_body(kind, record_best, rule)

    def _try_capture(self, key, body):
        """Capture `body` as graph `key`; a failed capture (driver / allocator state) falls back to eager launches."""
        try:
            g, n = self._capture(body)
        except Exception as e:      # nothing was executed during the capture: the device state is still the pre-capture one
            import warnings
            warnings.warn(f"coda_b200: CUDA graph capture failed ({type(e).__name__}: {e}); continuing with eager launches")
            self.use_graph = False
            self.pending, self.scored, self.reported = False, False, False
            torch.cuda.synchronize(self.dev)
            return None, 0
        self.graphs[key] = g
        return g, n

    def loop_capture(self, record_best: bool = False, rule: str = "first", kind: str = "eig"):
        key = ("loop", kind, bool(record_best), rule)
        with self._on():
            _g, self.loop_launches[key] = self._try_capture(key, lambda: self._loop_body(kind, record_best, rule))

    def loop_replay(self, k: int = 1, record_best: bool = False, rule: str = "first", kind: str = "eig"):
        key = ("loop", kind, bool(record_best), rule)
        with self._on():
            g = self.graphs.get(key)
            for _ in range(k):
                if g is None:
                    self._loop_body(kind, record_best, rule)
                else:
                    g.replay()
            if g is not None:
                self.counters["launches"] += k * self.loop_launches[key]

    # Buffers of the kinds other than "eig": the static scores (uncertainty), the candidates and the pre-draw rows.
    def abl_bind(self, kind, score=None, width=0, rows=0):
        with self._on():
            if kind == "uncertainty":
                if getattr(self, "abl_score", None) is None:
                    self.abl_score = score.to(self.dev, torch.float32).contiguous()
                return
            if getattr(self, "abl_cand", None) is None:
                self.abl_cand = self.disagree.to(torch.float32)
                self.abl_xp = self._z((2 * int(self.lib.coda_b200_select_blocks(self.N)),), torch.int64)
                self.abl_best = self._z((4,), torch.int64)
                self.abl_pick = self._z((1,), torch.int64)
                self.abl_lw = self._z((8,), torch.int64)
                self.abl_pre, self.abl_width, self.abl_recs, self.abl_nrec = None, 0, None, 0
            if self.abl_pre is None or self.abl_width != width or self.abl_pre.numel() != rows * width:
                self.abl_pre = self._z((rows * width,), torch.int64)
                self.abl_width = width
                if kind == "prefilter":
                    self.abl_nrec = int(self.lib.coda_b200_prefilter_blocks(width - 1))
                    self.abl_recs = self._z((4 * self.abl_nrec,), torch.int64)
                drawn = ("iid", "prefilter", "prefilter_id")             # the graphs that read the old buffer
                for key in [k for k in self.graphs if isinstance(k, tuple) and k[1] in drawn]:
                    del self.graphs[key]

    def abl_load(self, pre_host):
        """Pre-draw rows (pinned int64, row-major) -> the device buffer; the next step reads row 0."""
        with self._on():
            self.abl_pre[: pre_host.numel()].copy_(pre_host, non_blocking=True)
            self.abl_lw[0:1].zero_()

    # ---- tie_rule="reference": a replica of Python's generator on this shard (csrc/pyrandom.cuh) --------------------
    # pyrng [625] int32 (the uint32 words of random.getstate()[1]); ref_lw [8] int64 loop words of the reference-mode
    # kernels: [0] pre row, [3] the pending word, [4] the prefilter winner's EIG bits; ref_xp: tie_band's partials.
    def ref_bind(self):
        with self._on():
            if getattr(self, "pyrng", None) is None:
                self.pyrng = self._z((625,), torch.int32)
                self.ref_lw = self._z((8,), torch.int64)
                self.ref_xp = self._z((2 * int(self.lib.coda_b200_select_blocks(self.N)),), torch.int64)

    def ref_bind_prefilter(self, m, setsize):
        """Scratch of the device sampler and of the prefilter's tie draw for prefilter_n = m (abl_bind first)."""
        with self._on():
            if getattr(self, "ref_m", None) != (m, setsize):
                self.ref_m, self.ref_setsize = (m, setsize), int(setsize)
                self.ref_pool = self._z((min(int(setsize), self.n_global) + 1,), torch.int32)
                self.ref_seen = self._z(((self.n_global + 31) // 32 + 1,), torch.int32)
                self.ref_band = self._z((m,), torch.int64)
                self.ref_bits = self._z(((m + 127) // 128 * 4,), torch.int32)

    def rng_upload(self, words):
        """words: CPU int32 [625] -> this shard's replica (ordered on its stream)."""
        with self._on():
            self.pyrng.copy_(words)

    def rng_download(self):
        with self._on():
            return self.pyrng.cpu()

    def candidate_counts(self):
        """(unlabeled items some model disagrees on, unlabeled items) of this shard; synchronises."""
        with self._on():
            un = self.labeled == 0
            return int((un & (self.disagree != 0)).sum()), int(un.sum())

    def _capture(self, body):
        torch.cuda.synchronize(self.dev)
        g = torch.cuda.CUDAGraph()
        cap_stream = self.stream or torch.cuda.Stream(device=self.dev)
        before = self.counters["launches"]
        if self.pending:                                        # join eager side-stream work before the capture starts
            self._cur().wait_event(self.ev_join)
            self.pending = False
        self.scored = False
        with torch.cuda.graph(g, stream=cap_stream, capture_error_mode="relaxed"):
            body()
            if self.pending:                                    # every forked stream has to rejoin inside the capture
                self._cur().wait_event(self.ev_join)
                self.pending = False
        launches = self.counters["launches"] - before
        self.counters["launches"] = before
        torch.cuda.synchronize(self.dev)
        return g, launches

    # ------------------------------------------------------------------------ API path
    def _report(self):
        """coda.py:306-309: global record + isclose tie list of every shard -> pinned host block (enqueue only)."""
        self._score()
        N, s = self.N, self._s()
        self._call("coda_b200_step_merge", self.st, self._x(), s)
        self._call("coda_b200_ties", _ptr(self.eig), N, _ptr(self.labeled), _ptr(self.disagree), self.n_offset,
                   _ptr(self.bestrec), TIE_CAP, _ptr(self.tie_hdr), _ptr(self.tie_idx), _ptr(self.tie_val), s, n=2)
        self._call("coda_b200_report_gather", _ptr(self.rep), REP_WORDS, _ptr(self.rep_all), self._x(), _ptr(self.flags), s)
        self.rep_host.copy_(self.rep_all, non_blocking=True)
        self.reported = True

    def report(self):
        with self._on():
            if not self.reported:
                self._report()

    def _api_body(self):
        self._call("coda_b200_step_label", self.st, self._x(), self._s())
        self._post_label()
        self._report()

    # add_label in phases (a front end driving several shards calls each phase on every shard before the next, so
    # that nothing blocks the host -- a graph capture synchronises the device -- while a peer's kernels are missing):
    #   label_stage    stage the host-chosen (idx, class) record: pinned ring slot -> device, no exchange inside
    #   api_capture    (once, after two eager steps) capture label + refresh + scoring pass + report as one graph
    #   label_run      replay the graph, or enqueue the same kernels one by one
    def label_stage(self, idx_global: int, true_class: int):
        with self._on():
            k = self.sel_pos
            self.sel_pos = (k + 1) % len(self.sel_events)
            if self.sel_events[k] is not None:
                self.sel_events[k].synchronize()                # the copy that last used this slot has executed
            loc = idx_global - self.n_offset
            self.sel_ring[k, 0] = loc if 0 <= loc < self.N else -1
            self.sel_ring[k, 1] = true_class
            self.sel.copy_(self.sel_ring[k], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self._cur())
            self.sel_events[k] = ev

    def api_graph_wanted(self) -> bool:
        return (self.use_graph and self.graphs.get("api") is None and self.graphs.get("api_warm", 0) >= 2
                and (self.cache_valid or self.mode != "incremental"))

    def api_capture(self):
        with self._on():
            _g, self.launches_per_api_step = self._try_capture("api", self._api_body)

    def label_run(self, eager_report: bool = True):
        with self._on():
            if not eager_report:
                self._call("coda_b200_step_label", self.st, self._x(), self._s())
                self._post_label()
                return
            g = self.graphs.get("api") if self.use_graph else None
            if g is not None:
                if self.pending:
                    self._cur().wait_event(self.ev_join)
                    self.pending = False
                g.replay()
                self.counters["launches"] += self.launches_per_api_step
                self.scored, self.reported = True, True
                return
            self.graphs["api_warm"] = self.graphs.get("api_warm", 0) + 1
            self._api_body()

    def label(self, idx_global: int, true_class: int, eager_report: bool = True):
        """coda.py:316-319 for a host-chosen (idx, class): stage the record, posterior update, marginal refresh and --
        so that the next get_next_item_to_label only has to wait -- the next scoring pass + report.  Enqueue only."""
        self.label_stage(idx_global, true_class)
        if eager_report and self.api_graph_wanted():
            self.api_capture()
        self.label_run(eager_report)

    def fetch(self):
        """Wait for the report block and decode it.  Returns a dict of host values."""
        with self._on():
            if not self.reported:
                self._report()
            self._cur().synchronize()
        allr = self.rep_host.numpy()                            # (world, REP_WORDS)
        r0 = allr[0]
        flags = 0
        for r in allr:
            flags |= int(r[0:1].view(np.int32)[0])
        use_a = int(r0[3]) > 0                                  # the record is the merged (global) one on every shard
        bits = int(r0[1] if use_a else r0[4])
        best_val = float(np.array([bits & 0xFFFFFFFF], dtype=np.uint32).view(np.float32)[0])
        n_ties = int(sum(int(r[9]) for r in allr))
        idxs, vals = [], []
        for r in allr:
            k = min(int(r[9]), TIE_CAP)
            idxs.append(r[12:12 + k])
            vals.append(r[12 + TIE_CAP:].view(np.float32)[:k])
        return dict(flags=flags, use_a=use_a, n_cand=int(r0[3]), best_val=best_val,
                    best_idx=int(r0[2] if use_a else r0[5]), n_ties=n_ties,
                    tie_min=int(min(int(r[10]) for r in allr)), tie_idx=np.concatenate(idxs).copy(),
                    tie_val=np.concatenate(vals).copy())

    def check_flags(self, sync=False, flags=None):
        if flags is None:
            flags = int(self.flags.item()) if sync else 0
        if not flags:
            return
        if flags & nat.FLAG_ROWSUM_WARN:                        # util.py:37-39 prints a warning and carries on
            print("[WARN] Pbest(beta) normalized rows not normalised")
            self.flags.bitwise_and_(~nat.FLAG_ROWSUM_WARN)
            flags &= ~nat.FLAG_ROWSUM_WARN
            if not flags:
                return
        if flags & nat.FLAG_PIPELINE_TIMEOUT:
            raise RuntimeError("coda_b200: the tensor-core marginal pass (k_pi_full_tc) stopped; its result is invalid")
        if flags & nat.FLAG_XCHG_TIMEOUT:
            raise RuntimeError("coda_b200: a shard did not arrive at an exchange within 2 s (peer crashed or not launched)")
        if flags & nat.FLAG_NO_CANDIDATE:
            raise RuntimeError("no unlabeled items left to select from")
        if flags & nat.FLAG_PREDRAW_MISMATCH:
            raise RuntimeError("coda_b200: a device-loop step found a candidate count other than the one its "
                               "pre-drawn random numbers were made for; the run does not follow the API path")
        if flags & nat.FLAG_NEGATIVE_PROB:
            raise RuntimeError("Pbest(beta) normalized has negatives")                 # util.py:33-35
        if flags & nat.FLAG_RANGE_INPUT and not flags & nat.FLAG_NONFINITE_INPUT:
            raise ValueError("coda_b200: dataset.preds must hold post-softmax scores in [0, 1] (coda/datasets.py:6)")
        names = [v for k, v in nat.FLAG_NAMES.items() if flags & k]
        raise RuntimeError(f"[NUMERIC ERROR] {', '.join(names)} has bad values (NaN/Inf)")   # util.py:20-25

    def mark_labeled(self, idx_global: int):
        loc = idx_global - self.n_offset
        with self._on():
            if 0 <= loc < self.N:
                self.labeled[loc] = 1
            self.scored = False
            self.reported = False

    # ------------------------------------------------------------------------- read-outs
    def pbest(self) -> torch.Tensor:
        with self._on():
            return self.m0[: self.H].clone().view(1, self.H)    # coda.py:329 -> (1, H)

    def pi_hat_xi(self) -> torch.Tensor:
        with self._on():
            xi = torch.empty_like(self.U)
            scratch = torch.zeros_like(self.pisum)
            self._call("coda_b200_pi_reduce", _ptr(self.U), self.N, self.C, self.fx_shift, _ptr(xi), _ptr(scratch),
                       _ptr(self.flags), self._s())
            return xi

    # ------------------------------------------------------------------------- checkpoint
    def state_tensors(self):
        """Everything a resumed run cannot rebuild from the slab alone (SURVEY.md 8f rank 4): the posterior, the
        un-normalised marginals they imply, the label mask and the device step counter."""
        return {"D": self.D, "U": self.U, "labeled": self.labeled, "pisum": self.pisum, "step_ctr": self.step_ctr}

    def __del__(self):
        try:
            _release_const_slot(self.dev.index, getattr(self, "const_slot", -1))
        except Exception:
            pass

    def close(self):
        """Release the graphs, the mailbox and every device buffer of this shard (the object is unusable afterwards)."""
        self.graphs.clear()
        _release_const_slot(self.dev.index, self.const_slot)
        self.const_slot = -1
        if self._mailbox is not None:
            self._mailbox.close()
            self._mailbox = None
        for k, v in list(self.__dict__.items()):
            if isinstance(v, torch.Tensor) or k in ("preds", "compact", "host", "host_slots", "st", "xchg", "_labels_keep",
                                                    "cidx"):
                setattr(self, k, None)


def build_engines(shards, group, **kw):
    """Construct the shards of one task in lock-step (``shards``: list of (preds, n_offset) on this process).
    Phase order matters once peers spin on each other: every shard enqueues its mixture before any host sync."""
    n_global = kw.pop("n_global")
    own = len(shards) > 1
    engines = [Engine(p, n_offset=off, n_global=n_global, world=group.world, own_stream=own, **kw) for p, off in shards]
    for e in engines:
        e.construct_scan()
    group.attach(engines)
    group.allreduce_sum_([e.conf_buf for e in engines])         # coda.py:42 sums over ALL items
    for e in engines:
        e.construct_posterior()
    # shadows last: every row cache of a device is in place before any shadow takes what is left, and shards that
    # share a device split what is left between them
    total = {}
    for e in engines:
        total[e.dev] = total.get(e.dev, 0) + 1
    left = dict(total)
    for e in engines:
        e.construct_tables(left[e.dev], total[e.dev])
        left[e.dev] -= 1
    for e in engines:
        e.construct_mixture()
    for e in engines:
        e.construct_finish()
    return engines
