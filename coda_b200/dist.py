"""N-axis sharding: who exchanges what, and how the shards reach each other's mailbox (SURVEY.md 8e).

Every shard owns a contiguous range of items and a replica of the small global state (dirichlets, tables,
pi_hat).  Per acquisition step exactly two exchanges cross GPUs, both INSIDE the fused step kernels
(``csrc/xchg.cuh``, ``csrc/step.cu``) as peer-memory stores over NVLink -- no NCCL call sits on the step path:

  1. arg-max     every shard stores {its best record, p_h(idx) of its best candidates} into every peer's mailbox;
                 all shards merge to the same global record and so know the chosen item AND its hard-prediction row
  2. marginals   every shard stores its sum_n pi_hat_xi[n, :] (int64 fixed point: exact, so pi_hat is
                 bit-identical for every shard count); all shards add them up in rank order

The API path (host picks / host labels) adds a third, the owner's p_h(idx) for a host-chosen idx, and ships the tie
lists the same way.  Construction adds one SUM all-reduce of the (H, C, C) soft-confusion sums (coda.py:42) -- bulk
data, so that one goes through NCCL (``TorchComm``) or, with one process driving all GPUs, through peer copies.

Two ways to form a group:
  ``ProcessGroup``    one process per GPU (torchrun): mailboxes are mapped with CUDA IPC handles
  ``InProcessGroup``  one Python process drives all shards (``main.py`` unchanged): plain peer access; the shards may
                      even share one GPU (each on its own stream), which is how the 1-GPU test tier covers sharding
"""
from __future__ import annotations

import ctypes as ct

import torch

from . import _native as nat
from .datasets import HostSlab, PieceSlab, piece_counts, piece_plan


class LocalComm:
    world = 1
    rank = 0

    def allreduce_sum_(self, t):
        return t

    def allreduce_min_(self, t):
        return t

    def allgather(self, t):
        return t.unsqueeze(0)

    def barrier(self):
        pass


class TorchComm:
    """torch.distributed process group (NCCL on GPUs, gloo in the CPU tests): construction-time reductions."""

    def __init__(self, group=None):
        import torch.distributed as dist
        if not dist.is_initialized():
            raise RuntimeError("torch.distributed is not initialised")
        self.dist = dist
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)

    def allreduce_sum_(self, t):
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM, group=self.group)
        return t

    def allreduce_min_(self, t):
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MIN, group=self.group)
        return t

    def allgather(self, t):
        out = torch.empty((self.world,) + tuple(t.shape), dtype=t.dtype, device=t.device)
        self.dist.all_gather_into_tensor(out.view(-1), t.contiguous().view(-1), group=self.group)
        return out

    def barrier(self):
        self.dist.barrier(group=self.group)


def preload_kernels() -> int:
    """Load every kernel of the library into the current device's context (once per device and process)."""
    d = torch.cuda.current_device()
    if d not in _PRELOADED:
        n = ct.c_int64(0)
        nat.check(nat.load().coda_b200_preload_kernels(ct.byref(n)), "preload_kernels")
        _PRELOADED[d] = int(n.value)
    return _PRELOADED[d]


_PRELOADED = {}


def default_comm():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return TorchComm()
    return LocalComm()


# ---------------------------------------------------------------------------------------
# mailboxes
# ---------------------------------------------------------------------------------------
class Mailbox:
    """One shard's mailbox (device memory from the library's own cudaMalloc, so it can be IPC-exported)."""

    def __init__(self, device, world, H, C, rep_words):
        self.lib = nat.load()
        self.device = torch.device(device)
        self.dims = (int(world), int(H), int(C), int(rep_words))
        self.bytes = int(self.lib.coda_b200_xchg_box_bytes(*self.dims))
        ptr = ct.c_void_p()
        with torch.cuda.device(self.device):
            nat.check(self.lib.coda_b200_xchg_alloc(self.bytes, ct.byref(ptr)), "xchg_alloc")
        self.ptr = int(ptr.value)
        self.epoch = torch.zeros(8, dtype=torch.int64, device=self.device)     # epochs [0..4), wait ns [4..8)
        torch.cuda.synchronize(self.device)     # the zero fill ran on the current stream; shards may use their own
        self.opened = []

    def export(self) -> bytes:
        buf = ct.create_string_buffer(64)
        with torch.cuda.device(self.device):
            nat.check(self.lib.coda_b200_ipc_export(self.ptr, buf), "ipc_export")
        return buf.raw

    def open_peer(self, handle: bytes) -> int:
        out = ct.c_void_p()
        with torch.cuda.device(self.device):
            nat.check(self.lib.coda_b200_ipc_open(ct.create_string_buffer(handle, 64), ct.byref(out)), "ipc_open")
        self.opened.append(int(out.value))
        return int(out.value)

    def view(self, rank, peer_ptrs) -> nat.XchgStruct:
        world, H, Cc, rep_words = self.dims
        x = nat.XchgStruct()
        x.world, x.rank = world, rank
        for r, ptr in enumerate(peer_ptrs):
            x.box[r] = ptr
        x.epoch = self.epoch.data_ptr()
        x.H, x.C, x.rep_words = H, Cc, rep_words
        return x

    def close(self):
        lib = self.lib
        try:
            with torch.cuda.device(self.device):
                for q in self.opened:
                    lib.coda_b200_ipc_close(q)
                self.opened = []
                if self.ptr:
                    lib.coda_b200_xchg_free(self.ptr)
                    self.ptr = 0
        except Exception:
            pass


def host_slab_refusals(gpus, shards, world):
    """What a host-resident slab (``HostSlab``) does not offer: it runs as one shard on one GPU in one process."""
    if (gpus and int(gpus) > 1) or (shards and int(shards) > 1) or world > 1:
        raise NotImplementedError("coda_b200: a HostSlab runs as one shard on one GPU (gpus=1, shards=1, one process); "
                                  "load the task as per-GPU pieces (ShardedHostSlab, ShardedSlab) to use several "
                                  "GPUs")


def piece_layout(slab, gpus, shards, world):
    """A ``PieceSlab`` (``ShardedSlab``, ``ShardedCompactSlab``, ``ShardedHostSlab``) is its own shard layout:
    [(piece, n_offset)], used in place (no peer copy, no re-split, and ``CODA_B200_GPUS`` is not consulted).
    ``shards=`` (or ``gpus=`` alone) must equal the piece count, ``gpus=`` with ``shards=`` the number of devices the
    pieces are on."""
    name = type(slab).__name__
    if world > 1:
        raise ValueError(f"coda_b200: a {name} holds the whole task in one process; under torch.distributed with "
                         "world > 1 every rank passes its own N-range tensor (e.g. ShardedFileDataset)")
    k = len(slab.pieces)
    want = shards or gpus
    if want and int(want) != k:
        raise ValueError(f"coda_b200: the {name} has {k} pieces, one shard each; "
                         f"{'shards' if shards else 'gpus'}={want} disagrees")
    ndev = len({p.device for p in slab.pieces})
    if shards and gpus and int(gpus) != ndev:
        raise ValueError(f"coda_b200: the {name}'s pieces are on {ndev} devices; gpus={gpus} disagrees")
    return slab.layout()


def shard_layout(preds, gpus, shards, comm, n_offset=0, default=lambda: 1):
    """-> (group, [(shard slab, n_offset)] of this process) of a selector over ``preds``:

    * a ``HostSlab``: one shard on its compute device;
    * a ``PieceSlab``: its pieces, one shard each (``piece_layout``);
    * a tensor or ``CompactSlab`` under torch.distributed with world > 1: this rank's shard of the task;
    * else a tensor or ``CompactSlab`` split into ``piece_counts`` N-range shards (``default()`` when neither
      ``shards=`` nor ``gpus=`` is given), or kept whole as one."""
    if isinstance(preds, HostSlab):
        host_slab_refusals(gpus, shards, comm.world)
        return SoloGroup(), [(preds, 0)]
    if isinstance(preds, PieceSlab):
        layout = piece_layout(preds, gpus, shards, comm.world)
        return (SoloGroup() if len(layout) == 1 else InProcessGroup(len(layout))), layout
    if comm.world > 1:
        return ProcessGroup(comm), [(preds, n_offset)]
    nshards, ngpus = piece_counts(preds.shape[1], shards, gpus, default)
    if nshards == 1:
        return SoloGroup(), [(preds, n_offset)]
    return InProcessGroup(nshards), split_slab(preds, nshards, ngpus)


def split_slab(preds, nshards, ngpus):
    """N-range shards of a slab that lives on one device, as ``datasets.piece_plan`` places them -> [(shard slab,
    n_offset)]: shards on the home device are VIEWS of the caller's tensor (the kernels take the model stride), the
    others are contiguous copies on their device.  Works for a dense tensor and a ``CompactSlab``."""
    home = preds.device.index
    plan = piece_plan(preds.shape[1], nshards, ngpus, home, torch.cuda.device_count())
    out = []
    for lo, hi, d in plan:
        if isinstance(preds, torch.Tensor):
            view = preds[:, lo:hi]
            if d != home:
                view = view.to(torch.device("cuda", d)).contiguous()
        else:                                           # CompactSlab
            view = preds.narrow_items(lo, hi)
            if d != home:
                view = view.to(torch.device("cuda", d))
        out.append((view, lo))
    for d in {d for _, _, d in plan}:                   # the peer copies ran on the current streams; the shards use their own
        torch.cuda.synchronize(d)
    return out


def labels_per_device(labels, devices):
    """{device: ``labels`` as a contiguous int64 tensor there} for the host-free loops, one copy per distinct device.
    Each device is synchronised once: the copies ran on the current streams, the shards read them on their own."""
    per_dev = {}
    for d in devices:
        if d not in per_dev:
            per_dev[d] = labels.to(d, torch.int64).contiguous()
    for d in per_dev:
        torch.cuda.synchronize(d)
    return per_dev


class SoloGroup:
    """world == 1: no exchange."""
    world = 1

    def __init__(self):
        self.comm = LocalComm()

    def rank_of(self, engine):
        return 0

    def attach(self, engines):
        for e in engines:
            e.xchg = None

    def allreduce_sum_(self, tensors):
        return tensors

    def barrier(self):
        pass


class ProcessGroup:
    """One process per GPU (torchrun).  ``comm`` does the construction-time all-reduce; mailboxes go through CUDA IPC."""

    def __init__(self, comm: TorchComm):
        self.comm = comm
        self.world, self.rank = comm.world, comm.rank
        self.box = None

    def rank_of(self, engine):
        return self.rank

    def attach(self, engines):
        (eng,) = engines
        self.box = Mailbox(eng.dev, self.world, eng.H, eng.C, eng.rep_words)
        mine = torch.frombuffer(bytearray(self.box.export()), dtype=torch.uint8).to(eng.dev)
        allh = self.comm.allgather(mine).cpu()                               # (world, 64)
        ptrs = []
        for r in range(self.world):
            ptrs.append(self.box.ptr if r == self.rank else self.box.open_peer(bytes(allh[r].numpy().tobytes())))
        eng.xchg = self.box.view(self.rank, ptrs)
        eng._mailbox = self.box
        self.comm.barrier()                                                  # every mailbox exists and is zeroed

    def allreduce_sum_(self, tensors):
        for t in tensors:
            self.comm.allreduce_sum_(t)
        return tensors

    def barrier(self):
        self.comm.barrier()


class InProcessGroup:
    """All shards driven by this process: engines[r] is rank r, on any mix of devices (peer access is enabled
    between distinct devices; shards on the same device just use different streams)."""

    def __init__(self, world):
        self.world = int(world)
        self.comm = LocalComm()
        self.boxes = []
        self._engines = []

    def rank_of(self, engine):
        return self._engines.index(engine)

    def attach(self, engines):
        assert len(engines) == self.world
        self._engines = list(engines)
        lib = nat.load()
        devs = sorted({e.dev.index for e in engines})
        for d in devs:                      # before any exchange kernel spins (csrc/preload.cu): no first-launch load waits
            with torch.cuda.device(d):      # for a peer that is waiting for this shard
                preload_kernels()
        for a in devs:
            for b in devs:
                if a != b:
                    with torch.cuda.device(a):
                        nat.check(lib.coda_b200_peer_enable(b), "peer_enable")
        self.boxes = [Mailbox(e.dev, self.world, e.H, e.C, e.rep_words) for e in engines]
        ptrs = [b.ptr for b in self.boxes]
        for r, e in enumerate(engines):
            e.xchg = self.boxes[r].view(r, ptrs)
            e._mailbox = self.boxes[r]

    def allreduce_sum_(self, tensors):
        """tensors[r] lives on engine r's device: every one ends up holding the sum (construction only)."""
        for t, e in zip(tensors, self._engines):
            e.sync()
        tot = tensors[0].clone()
        for t in tensors[1:]:
            tot += t.to(tot.device)
        for t in tensors:
            t.copy_(tot.to(t.device))
        for d in {t.device for t in tensors}:
            torch.cuda.synchronize(d)
        return tensors

    def barrier(self):
        pass


# ---------------------------------------------------------------------------------------
# host-side mirrors of the device merge rules (used by the CPU/gloo tests and the slow paths)
# ---------------------------------------------------------------------------------------
IDX_NONE = (1 << 63) - 1


def merge_records(recs):
    """recs: iterable of (vA, iA, cntA, vB, iB).  Max value, lowest index on equal values,
    counts summed -- the rule of best2_merge (csrc/common.cuh) without the runner-up."""
    va, ia, ca, vb, ib = float("-inf"), IDX_NONE, 0, float("-inf"), IDX_NONE
    for (a, i, c, b, j) in recs:
        if a > va or (a == va and i < ia):
            va, ia = a, i
        if b > vb or (b == vb and j < ib):
            vb, ib = b, j
        ca += c
    return va, ia, ca, vb, ib


def merge_best2(items):
    """Host mirror of best2_merge: items = iterable of (v, i, v2); returns the merged (v, i, v2) where v2 is the
    best value among all OTHER items (the runner-up the isclose tie test needs)."""
    v, i, v2 = float("-inf"), IDX_NONE, float("-inf")
    for (ov, oi, ov2) in items:
        if oi == IDX_NONE:
            continue
        if i == IDX_NONE:
            v, i, v2 = ov, oi, ov2
        elif ov > v or (ov == v and oi < i):
            v2 = max(v2, ov2, v)
            v, i = ov, oi
        else:
            v2 = max(v2, ov2, ov)
    return v, i, v2


def choose_among_ties(tie_idx, rng):
    """coda.py:308: random.choice over the tied candidates in ascending index order.  ``random.choice``
    consumes exactly one ``_randbelow(len)``, so choosing a position is RNG-equivalent."""
    order = sorted(int(i) for i in tie_idx)
    return order[rng.choice(range(len(order)))]


# host mirrors of the competing selectors' shard merges (csrc/baselines.cu, the *_xchg entry points)
def merge_extreme(recs, want_max, rank):
    """recs: per-shard (value, count) in rank order (count 0 = no unlabeled item on that shard).  -> (value, global count,
    ties on ranks below ``rank``, ties on ``rank``): the rule of k_extreme_xchg."""
    v, n = 0.0, 0
    for (b, c) in recs:
        if c == 0:
            continue
        if n == 0 or (b > v if want_max else b < v):
            v, n = b, c
        elif b == v:
            n += c
    tied = [c if (n > 0 and c > 0 and b == v) else 0 for (b, c) in recs]
    return v, n, sum(tied[:rank]), tied[rank]


def kth_owner(recs, want_max, k):
    """The shard whose ties cover the k-th tied item (k_select_kth_xchg) and the item's rank among that shard's ties."""
    for r in range(len(recs)):
        _v, _n, lower, mine = merge_extreme(recs, want_max, r)
        if lower <= k < lower + mine:
            return r, k - lower
    return -1, -1


def draw_owner(sums, counts, u):
    """k_wdraw_xchg's first merge: per-shard sums of the normalised weights and unlabeled counts in rank order ->
    (owner shard, running sum and position before it, target = u * grand total), the last non-empty shard when rounding
    leaves the target at or beyond the total; (-1, 0, 0, target) when no item is unlabeled."""
    grand = 0.0
    for s in sums:
        grand += s
    target = u * grand
    base, pos, owner, last = 0.0, 0, -1, -1
    for r, (s, c) in enumerate(zip(sums, counts)):
        if c == 0:
            continue
        last = r
        if base + s > target:
            owner = r
            break
        base += s
        pos += c
    if owner < 0 and last >= 0:
        owner = last
        base -= sums[last]
        pos -= counts[last]
    return owner, base, pos, target
