"""Datasets: the reference loader contract (coda/datasets.py:4-23) plus shard-aware variants."""
from __future__ import annotations

import ctypes as ct
import functools
import os

import torch

from .synth import shard_range, synth, synth_compact


_KEPT_DTYPES = (torch.float32, torch.float16, torch.bfloat16)


def _slab_dtype(t: torch.Tensor, keep_dtype: bool) -> torch.dtype:
    """fp32 (coda/datasets.py:14 widens on load), or with ``keep_dtype`` the stored width of an fp16 / bf16 / fp32 slab:
    the kernels widen 16-bit values exactly, so the results are those of the fp32 slab at half the memory."""
    return t.dtype if keep_dtype and t.dtype in _KEPT_DTYPES else torch.float32


class PieceSlab:
    """An (H, N, C) slab held as contiguous N-range pieces, each on its own device (consecutive pieces may share one).
    The pieces ARE the shard layout: CODA and the competing selectors run one shard per piece, in place.  Duck-types the
    tensor attributes the selectors and main.py read from ``dataset.preds``; ``device`` is the first piece's.  The
    subclasses check their pieces (``_check``)."""

    def __init__(self, pieces):
        pieces = list(pieces)
        if not pieces:
            raise ValueError(f"{type(self).__name__}: at least one piece expected")
        self._check(pieces)
        H, _, C = pieces[0].shape
        self.pieces = pieces
        self.offsets = []
        n = 0
        for p in pieces:
            self.offsets.append(n)
            n += int(p.shape[1])
        self.shape = torch.Size([int(H), n, int(C)])
        self.device = pieces[0].device
        self.dtype = pieces[0].dtype
        self.is_cuda = pieces[0].is_cuda

    def layout(self):
        """[(piece, n_offset)]: the shard layout selectors build from."""
        return list(zip(self.pieces, self.offsets))

    def numel(self):
        return self.shape[0] * self.shape[1] * self.shape[2]

    def element_size(self):
        return self.pieces[0].element_size()

    def item_column(self, idx) -> torch.Tensor:
        """The (H, C) float32 scores of item ``idx``, on the (compute) device of the piece that holds it."""
        idx = int(idx)
        if not 0 <= idx < self.shape[1]:
            raise IndexError(f"{type(self).__name__}: item {idx} outside [0, {self.shape[1]})")
        r = max(i for i, off in enumerate(self.offsets) if off <= idx)
        p, i = self.pieces[r], idx - self.offsets[r]
        return p[:, i].float() if isinstance(p, torch.Tensor) else p.item_column(i)


def pieces_of(preds):
    """[(piece, n_offset)] of a slab: a ``PieceSlab``'s pieces, else the slab itself as one piece."""
    return preds.layout() if isinstance(preds, PieceSlab) else [(preds, 0)]


class ShardedSlab(PieceSlab):
    """A ``PieceSlab`` of dense (H, N_i, C) tensors."""

    @staticmethod
    def _check(pieces):
        for p in pieces:
            if isinstance(p, CompactSlab) or not isinstance(p, torch.Tensor):
                raise TypeError("ShardedSlab: pieces must be dense (H, N_i, C) tensors; a compact ShardedSlab is not "
                                "supported")
            if p.dim() != 3 or p.dtype not in _KEPT_DTYPES:
                raise TypeError(f"ShardedSlab: pieces must be float32, float16 or bfloat16 (H, N_i, C) tensors, got "
                                f"{p.dtype} {tuple(p.shape)}")
            if not p.is_contiguous() or p.shape[1] < 1:
                raise ValueError("ShardedSlab: every piece must be a contiguous tensor with at least one item")
        H, _, C = pieces[0].shape
        if any(p.shape[0] != H or p.shape[2] != C or p.dtype != pieces[0].dtype for p in pieces):
            raise TypeError("ShardedSlab: all pieces must share one dtype, H and C")


HOST_CHUNK_BYTES = 1 << 30
HOST_CHUNK_ALIGN = 32           # items: a multiple of the slab scan's tile, so a chunk takes the scan the whole slab takes


class HostSlab:
    """An (H, N, C) slab kept in host memory -- a contiguous CPU tensor, possibly memory-mapped from a ``torch.save``
    file, or an N-range view of one (each model's items one contiguous range) -- for one compute ``device``: a task
    larger than one GPU, run exactly on that GPU.  CODA, the competing selectors and ``Oracle.true_losses`` stream it
    through the device in N-range chunks of ``chunk_items`` items (two device buffers of one chunk each); the slab is
    never copied whole to the device.  Duck-types ``ShardedSlab``'s surface: ``shape``, ``dtype`` (the width the
    kernels read: the tensor's, or float32 to widen a 16-bit tensor on the device), ``device``, ``numel``,
    ``element_size``, ``item_column``."""

    def __init__(self, preds: torch.Tensor, device, dtype=None, chunk_items=None):
        if not isinstance(preds, torch.Tensor) or preds.device.type != "cpu":
            raise TypeError("HostSlab: a CPU (H, N, C) tensor expected")
        if preds.dim() != 3 or preds.dtype not in _KEPT_DTYPES:
            raise TypeError(f"HostSlab: a float32, float16 or bfloat16 (H, N, C) tensor expected, got {preds.dtype} "
                            f"{tuple(preds.shape)}")
        H, N, C = (int(s) for s in preds.shape)
        if N < 1 or not (preds.stride(2) == 1 and preds.stride(1) == C and (H == 1 or preds.stride(0) >= N * C)):
            raise ValueError("HostSlab: the tensor must hold at least one item, with contiguous items (a contiguous "
                             "tensor or an N-range view of one)")
        dtype = preds.dtype if dtype is None else dtype
        if dtype not in (preds.dtype, torch.float32):
            raise TypeError(f"HostSlab: a {preds.dtype} slab is read as {preds.dtype} or widened to float32, not {dtype}")
        self.host = preds
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise TypeError("HostSlab: the compute device must be a CUDA device")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.is_cuda = True
        self.dtype = dtype
        self.shape = torch.Size([H, N, C])
        if chunk_items is None:
            chunk_items = HOST_CHUNK_BYTES // (H * C * self.element_size())
        a = HOST_CHUNK_ALIGN
        self.chunk_items = min(max(a, (int(chunk_items) + a - 1) // a * a), (N + a - 1) // a * a)

    def numel(self):
        return self.shape[0] * self.shape[1] * self.shape[2]

    def element_size(self):
        return torch.empty(0, dtype=self.dtype).element_size()

    def chunk_bytes(self):
        """Device bytes of one chunk buffer."""
        return self.shape[0] * self.chunk_items * self.shape[2] * self.element_size()

    def item_column(self, idx) -> torch.Tensor:
        """The (H, C) float32 scores of item ``idx`` on the compute device."""
        idx = int(idx)
        if not 0 <= idx < self.shape[1]:
            raise IndexError(f"HostSlab: item {idx} outside [0, {self.shape[1]})")
        return self.host[:, idx].to(self.device).float()

    def walk(self, body, lo=0, hi=None):
        """Stream items [lo, hi) through the device: ``body(n0, n1, view)`` enqueues, on the current stream, the kernels
        that read ``view``, a contiguous (H, n1 - n0, C) device tensor at ``dtype`` holding items [n0, n1).  Each
        model's range is read from the host tensor through two pinned chunks (``_fill_device``); chunk i + 1 is copied
        into the second device buffer while the kernels of chunk i run.  Returns when every body's kernels are done."""
        H, N, C = self.shape
        hi = N if hi is None else hi
        step = self.chunk_items
        nb = min(2, (hi - lo + step - 1) // step)
        cur = torch.cuda.current_stream(self.device)
        bufs = [torch.empty(H * min(step, hi - lo) * C, dtype=self.dtype, device=self.device) for _ in range(nb)]
        used = [None] * nb
        for i, n0 in enumerate(range(lo, hi, step)):
            n1, j = min(hi, n0 + step), i % nb
            if used[j] is not None:
                used[j].synchronize()                              # the kernels that last read this buffer are done
            view = bufs[j][: H * (n1 - n0) * C].view(H, n1 - n0, C)
            _fill_device(self.host, [(view, n0, n1)], self.dtype, DEFAULT_CHUNK_BYTES)
            body(n0, n1, view)
            used[j] = torch.cuda.Event()
            used[j].record(cur)
        for ev in used:
            if ev is not None:
                ev.synchronize()


class HostDataset:
    """``dataset`` wrapper of a ``HostSlab`` for callers that already hold the CPU tensor (``labels`` on the device)."""

    def __init__(self, slab: HostSlab, labels=None):
        self.preds, self.labels, self.device = slab, labels, slab.device
        self.n_offset, self.n_global = 0, slab.shape[1]


class ShardedHostSlab(PieceSlab):
    """A ``PieceSlab`` kept in host memory, one ``HostSlab`` per piece, each computed on its own device: the
    host-resident twin of ``ShardedSlab``.  CODA and the competing selectors run one host-resident shard per piece, each
    streaming its piece through its own device and staging its own host columns each step, and give the bits of the
    whole slab."""

    @staticmethod
    def _check(pieces):
        for p in pieces:
            if not isinstance(p, HostSlab):
                raise TypeError("ShardedHostSlab: pieces must be HostSlab (device pieces make a ShardedSlab)")
        H, _, C = pieces[0].shape
        if any(p.shape[0] != H or p.shape[2] != C or p.dtype != pieces[0].dtype for p in pieces):
            raise TypeError("ShardedHostSlab: all pieces must share one dtype, H and C")


def walk(preds, body):
    """Read a dense piece on its device: ``body(n0, n1, view)`` enqueues the kernels that read ``view``, an
    (H, n1 - n0, C) device tensor holding items [n0, n1).  A ``HostSlab`` streams through its device in chunks
    (``HostSlab.walk``, which returns when they are done); a device tensor is one view of itself."""
    if isinstance(preds, HostSlab):
        preds.walk(body)
    else:
        body(0, int(preds.shape[1]), preds)


def model_stride(v):
    """Elements between two models' rows of an (H, n, C) view with contiguous items, as the slab kernels take it."""
    H, n, C = v.shape
    return int(v.stride(0)) if H > 1 else int(n) * int(C)


def load_host(filepath, device, keep_dtype=False, chunk_items=None, *, shards=None, gpus=None):
    """``filepath``'s (H, N, C) slab as a ``HostSlab`` over its memory map: a 16-bit file is read at its width with
    ``keep_dtype``, else widened to fp32 on the device chunk by chunk.  With ``shards=`` / ``gpus=``, a
    ``ShardedHostSlab`` of N-range views of that one memory map, with the ranges and devices of ``load_sharded``:
    nothing is copied on the host, and each piece streams through its own device."""
    full = _open_mmap(filepath)
    dtype = _slab_dtype(full, keep_dtype)
    if not (shards or gpus):
        return HostSlab(full, device, dtype=dtype, chunk_items=chunk_items)
    plan = _load_plan(int(full.shape[1]), torch.device(device), shards, gpus)
    return ShardedHostSlab([HostSlab(full[:, lo:hi], torch.device("cuda", d), dtype=dtype, chunk_items=chunk_items)
                            for lo, hi, d in plan])


def piece_plan(N, nshards, ngpus, home, device_count):
    """[(lo, hi, device index)] of ``nshards`` N-range pieces over ``ngpus`` devices, as the loaders and
    ``dist.split_slab`` make them: the ranges ``shard_range(N, r, nshards)``, the home device first, then the others in
    order, consecutive pieces sharing a device when there are more pieces than GPUs."""
    devs = [home] + [d for d in range(device_count) if d != home]
    devs = devs[:max(1, ngpus)]
    return [(*shard_range(N, r, nshards), devs[r * len(devs) // nshards]) for r in range(nshards)]


def piece_counts(N, shards, gpus, default=lambda: 1):
    """(pieces, GPUs) of a task of N items split by ``shards=`` / ``gpus=``: ``shards`` pieces (else ``gpus``, else
    ``default()``, at most N) over ``gpus`` GPUs (else as many as there are pieces, up to the visible GPUs)."""
    nshards = int(shards) if shards else (int(gpus) if gpus else int(default()))
    ngpus = int(gpus) if gpus else min(nshards, max(1, torch.cuda.device_count()))
    return max(1, min(nshards, N)), ngpus


def _load_plan(N, device, shards, gpus):
    """``piece_plan`` of a load split by ``shards=`` / ``gpus=`` (``piece_counts``), the first piece on ``device``."""
    nshards, ngpus = piece_counts(N, shards, gpus)
    home = device.index if device.index is not None else torch.cuda.current_device()
    return piece_plan(N, nshards, ngpus, home, torch.cuda.device_count())


def chunk_walk(lo, hi, C, esz, chunk_bytes):
    """[(a, b)] element ranges of one model's items [lo, hi) (the elements [lo*C, hi*C) of that model), at most
    ``chunk_bytes`` each (at least one element)."""
    step = max(1, int(chunk_bytes) // int(esz))
    a, end = lo * C, hi * C
    out = []
    while a < end:
        out.append((a, min(end, a + step)))
        a = out[-1][1]
    return out


DEFAULT_CHUNK_BYTES = 64 << 20


def _open_mmap(filepath):
    import zipfile
    if not zipfile.is_zipfile(filepath):
        raise ValueError(f"{filepath}: a sharded load memory-maps the file, which needs torch.save's zip format; this "
                         f"file is in the legacy format -- re-save it with torch.save(torch.load(path), path)")
    full = torch.load(filepath, map_location="cpu", mmap=True, weights_only=True)
    if not isinstance(full, torch.Tensor) or full.dim() != 3:
        raise ValueError(f"{filepath}: expected an (H, N, C) tensor")
    if not full.is_contiguous():
        raise ValueError(f"{filepath}: the saved (H, N, C) tensor is not contiguous, so a model's items are not one "
                         f"contiguous range of the file; re-save it with torch.save(t.contiguous(), path)")
    return full


def _fill_device(full, todo, dtype, chunk_bytes):
    """Fill the pieces ``todo`` = [(piece, lo, hi)] of one device model by model: each model's range is one contiguous
    read of the file, staged through two pinned chunks; a 16-bit file read into fp32 pieces is widened on the device.
    ``full`` is an (H, N, C) tensor with contiguous items: the file, or an N-range view of it."""
    dev = todo[0][0].device
    H, _, C = full.shape
    src_t = full.dtype
    esz = full.element_size()
    step = max(1, int(chunk_bytes) // esz)
    pins = [torch.empty(step, dtype=src_t, pin_memory=True) for _ in range(2)]
    done = [None, None]
    with torch.cuda.device(dev):
        stream = torch.cuda.Stream(device=dev)
        stage = torch.empty(step, dtype=src_t, device=dev) if src_t != dtype else None
        k = 0
        with torch.cuda.stream(stream):
            for piece, lo, hi in todo:
                dst = piece.view(H, -1)
                for h in range(H):
                    src = full[h].view(-1)                      # one model's items: contiguous
                    for a, b in chunk_walk(lo, hi, C, esz, chunk_bytes):
                        j = k % 2
                        if done[j] is not None:
                            done[j].synchronize()             # the copy that last read this pinned chunk is over
                        n = b - a
                        pins[j][:n].copy_(src[a:b])
                        out = dst[h, a - lo * C:b - lo * C]
                        if stage is None:
                            out.copy_(pins[j][:n], non_blocking=True)
                        else:
                            stage[:n].copy_(pins[j][:n], non_blocking=True)
                            out.copy_(stage[:n])                # fp16 / bf16 -> fp32 is exact
                        done[j] = torch.cuda.Event()
                        done[j].record(stream)
                        k += 1
        stream.synchronize()
        del stage


def load_sharded(filepath, device, keep_dtype=False, shards=None, gpus=None, chunk_bytes=DEFAULT_CHUNK_BYTES):
    """``filepath``'s (H, N, C) slab as a ``ShardedSlab`` of ``shards`` pieces over ``gpus`` devices, read through a
    memory map: no device ever holds more than its pieces plus one staging chunk, and host memory holds two pinned
    chunks per device.  Every piece equals ``torch.load(filepath)[:, lo:hi]`` at the slab dtype (see ``Dataset``)."""
    import concurrent.futures as cf
    full = _open_mmap(filepath)
    H, N, C = (int(s) for s in full.shape)
    dtype = _slab_dtype(full, keep_dtype)
    plan = _load_plan(N, torch.device(device), shards, gpus)
    pieces, by_dev = [], {}
    for lo, hi, d in plan:
        p = torch.empty((H, hi - lo, C), dtype=dtype, device=torch.device("cuda", d))
        pieces.append(p)
        by_dev.setdefault(d, []).append((p, lo, hi))
    with cf.ThreadPoolExecutor(max_workers=len(by_dev)) as ex:     # one host thread per device
        for f in [ex.submit(_fill_device, full, todo, dtype, chunk_bytes) for todo in by_dev.values()]:
            f.result()
    return ShardedSlab(pieces)


def _free_bytes(index):
    return torch.cuda.mem_get_info(index)[0]


def _map_contents(filepath):
    """``torch.load`` of a zip file through a memory map; None for a legacy-format file or one it does not read."""
    import zipfile
    if not zipfile.is_zipfile(filepath):
        return None
    try:
        return torch.load(filepath, map_location="cpu", mmap=True, weights_only=True)
    except Exception:
        return None


def load_route(filepath, device, env=None):
    """The keyword arguments ``coda.datasets.Dataset`` loads ``filepath`` on ``device`` with, under the ``CODA_B200_*``
    settings in ``env`` (default ``os.environ``; an empty value counts as unset).  A slab counts at the width it would
    be held at; the file is opened once and each device's free memory read at most once.

    * A ``CompactSlab.save`` file, or any file with ``CODA_B200_COMPACT_K=K``: a compact load, in device pieces by the
      last rule below on its compact byte count.
    * ``CODA_B200_HOST_SLAB=1``: one ``HostSlab``; any other value turns the host rules off.
    * One GPU visible: a ``HostSlab`` when the slab exceeds the target device's free memory.
    * More than one GPU visible and ``CODA_B200_SHARD_LOAD`` unset: ``CODA_B200_GPUS`` host pieces (else one per
      visible GPU) when the slab exceeds the summed free memory of the devices they would use, a shared one counted
      once.
    * Device pieces, as many: with ``CODA_B200_SHARD_LOAD=1``, or with more than one GPU visible when the slab exceeds
      the target device's free memory.
    * Else the plain load.

    A file that cannot be memory-mapped (the legacy format) keeps the plain load; so does a failure to read free
    memory in the host rules, while in the device-piece rule it raises."""
    env = os.environ if env is None else env
    keep = env.get("CODA_B200_KEEP_DTYPE", "0") == "1"
    k = int(env["CODA_B200_COMPACT_K"]) if env.get("CODA_B200_COMPACT_K") else None
    dev = torch.device(device)
    ngpus = torch.cuda.device_count()
    free = functools.cache(_free_bytes)

    def home():
        return dev.index if dev.index is not None else torch.cuda.current_device()

    def piece_count():
        return max(1, int(env["CODA_B200_GPUS"])) if env.get("CODA_B200_GPUS") else max(1, ngpus)

    def device_pieces(held):
        count = piece_count()
        if env.get("CODA_B200_SHARD_LOAD", "0") == "1":
            return count
        if dev.type != "cuda" or ngpus < 2 or held is None:
            return 0
        return count if held > free(home()) else 0

    obj = _map_contents(filepath)
    try:
        comp = _compact_contents(obj, filepath)
        compact = comp is not None
    except ValueError:                                             # a compact file load_compact refuses, saying why
        comp, compact = None, True
    except Exception:
        comp, compact = None, False
    full = obj if isinstance(obj, torch.Tensor) and obj.dim() == 3 and obj.is_contiguous() else None
    if k or compact:
        held = (comp["ids"].numel() * 6 if comp is not None
                else int(full.shape[0]) * int(full.shape[1]) * k * 6 if full is not None else None)
        return {"compact_k": k, "shards": device_pieces(held) or None}
    held = full.numel() * torch.empty(0, dtype=_slab_dtype(full, keep)).element_size() if full is not None else None
    host = env.get("CODA_B200_HOST_SLAB")
    if host:
        if host == "1":
            return {"keep_dtype": keep, "host": True}
    elif dev.type == "cuda" and held is not None and ngpus == 1:
        try:
            if held > free(home()):
                return {"keep_dtype": keep, "host": True}
        except RuntimeError:                                       # no usable device: keep the plain load
            pass
    elif dev.type == "cuda" and held is not None and ngpus > 1 and not env.get("CODA_B200_SHARD_LOAD"):
        count = piece_count()
        try:
            if held > sum(free(d) for d in {d for _, _, d in _load_plan(int(full.shape[1]), dev, count, None)}):
                return {"keep_dtype": keep, "host": True, "shards": count}
        except RuntimeError:                                       # no usable device: keep the plain load
            pass
    shards = device_pieces(held)
    return {"keep_dtype": keep, "shards": shards} if shards else {"keep_dtype": keep}


# ---------------------------------------------------------------------------------------------------------------------
# compact slabs: built on the device from dense scores (csrc/compact_build.cu), saved and loaded as pieces
# ---------------------------------------------------------------------------------------------------------------------
COMPACT_FORMAT = "coda_b200.compact"
COMPACT_VERSION = 1
COMPACT_KS = (1, 2, 3, 4, 8)                    # the instantiated K of csrc/compact.cu and csrc/compact_build.cu


def row_walk(lo, hi, C, esz, chunk_bytes):
    """[(a, b)] item ranges covering [lo, hi) of one model: whole items of C elements of ``esz`` bytes, at most
    ``chunk_bytes`` of them per range, and at least one item."""
    step = max(1, int(chunk_bytes) // (int(C) * int(esz)))
    return [(a, min(hi, a + step)) for a in range(lo, hi, step)]


def _open_compact(filepath):
    """The memory-mapped contents of a ``CompactSlab.save`` file, or None for any other file."""
    import zipfile
    if not zipfile.is_zipfile(filepath):
        return None
    return _compact_contents(torch.load(filepath, map_location="cpu", mmap=True, weights_only=True), filepath)


def _compact_contents(obj, filepath):
    """``obj``, the contents of ``filepath``, if it is a compact slab this loader reads; None for any other file."""
    if not (isinstance(obj, dict) and obj.get("format") == COMPACT_FORMAT):
        return None
    if obj.get("version") != COMPACT_VERSION:
        raise ValueError(f"{filepath}: compact slab format version {obj.get('version')}, this loader reads "
                         f"{COMPACT_VERSION}")
    ids, probs = obj["ids"], obj["probs"]
    if (ids.dim() != 3 or ids.shape != probs.shape or ids.dtype != torch.int16 or probs.dtype != torch.float32
            or not ids.is_contiguous() or not probs.is_contiguous()):
        raise ValueError(f"{filepath}: a compact slab file holds contiguous (H, N, K) int16 ids and float32 probs")
    return obj


def is_compact_file(filepath):
    """True for a file written by ``CompactSlab.save``."""
    try:
        return _open_compact(filepath) is not None
    except ValueError:                                             # a compact file this loader refuses: say why there
        return True
    except Exception:                                              # not something torch.load(weights_only) reads
        return False


def _raise_input_flags(flags):
    from . import _native as nat
    if flags & nat.FLAG_NONFINITE_INPUT:
        raise RuntimeError("[NUMERIC ERROR] preds has bad values (NaN/Inf)")
    if flags & nat.FLAG_RANGE_INPUT:
        raise ValueError("coda_b200: dataset.preds must hold post-softmax scores in [0, 1] (coda/datasets.py:6)")


def _compact_launch(lib, src, fmt, model_stride, H, N, C, K, ids, probs, out_stride, dropped, flat, flags, stream):
    from . import _native as nat
    nat.check(lib.coda_b200_compact_build(ct.c_void_p(src), fmt, int(model_stride), int(H), int(N), int(C), int(K),
                                          ct.c_void_p(ids), ct.c_void_p(probs), int(out_stride), ct.c_void_p(dropped),
                                          ct.c_void_p(flat), ct.c_void_p(flags), ct.c_void_p(stream)),
              "compact_build")


def _check_k(K, C):
    if K is None or int(K) not in COMPACT_KS or not int(K) < int(C):
        raise ValueError(f"coda_b200: compact K must be one of {COMPACT_KS} and below C = {C}, got {K}")
    if int(C) > 4096:
        raise ValueError(f"coda_b200: compacting takes C <= 4096 classes, got {C}")
    return int(K)


def _compact_device(full, todo, K, chunk_bytes):
    """Compact the pieces ``todo`` = [(CompactSlab piece, lo, hi)] of one device from the memory-mapped dense slab
    ``full``, model by model: whole items are staged through two pinned chunks and one device chunk at the file's dtype,
    and the kernel writes from that chunk straight into the piece.  -> (dropped_max, flat_rows, flags) of this device."""
    from . import _native as nat
    lib = nat.load()
    dev = todo[0][0].device
    H, _, C = (int(s) for s in full.shape)
    esz = full.element_size()
    fmt = nat.slab_format(full.dtype)
    step = max(1, int(chunk_bytes) // (C * esz)) * C
    pins = [torch.empty(step, dtype=full.dtype, pin_memory=True) for _ in range(2)]
    done = [None, None]
    flat_src = full.view(H, -1)
    with torch.cuda.device(dev):
        stream = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(stream):
            stage = torch.empty(step, dtype=full.dtype, device=dev)
            dropped = torch.zeros(H, dtype=torch.float32, device=dev)
            flat = torch.zeros(H, dtype=torch.int64, device=dev)
            flags = torch.zeros(1, dtype=torch.int32, device=dev)
            k = 0
            for piece, lo, hi in todo:
                for h in range(H):
                    for a, b in row_walk(lo, hi, C, esz, chunk_bytes):
                        j = k % 2
                        if done[j] is not None:
                            done[j].synchronize()             # the copy that last read this pinned chunk is over
                        n = (b - a) * C
                        pins[j][:n].copy_(flat_src[h, a * C:b * C])
                        stage[:n].copy_(pins[j][:n], non_blocking=True)
                        _compact_launch(lib, stage.data_ptr(), fmt, n, 1, b - a, C, K,
                                        piece.ids[h, a - lo:].data_ptr(), piece.probs[h, a - lo:].data_ptr(), 0,
                                        dropped[h:].data_ptr(), flat[h:].data_ptr(), flags.data_ptr(),
                                        stream.cuda_stream)
                        done[j] = torch.cuda.Event()
                        done[j].record(stream)
                        k += 1
        stream.synchronize()
        del stage
    return dropped, flat, int(flags.item())


def _copy_compact_device(obj, todo):
    """Copy the pieces ``todo`` = [(CompactSlab piece, lo, hi)] of one device out of a memory-mapped compact file, one
    model's item range at a time."""
    dev = todo[0][0].device
    with torch.cuda.device(dev):
        for piece, lo, hi in todo:
            for h in range(piece.shape[0]):
                piece.ids[h].copy_(obj["ids"][h, lo:hi])
                piece.probs[h].copy_(obj["probs"][h, lo:hi])
        torch.cuda.synchronize(dev)


def load_compact(filepath, device, K=None, *, shards=None, gpus=None, chunk_bytes=DEFAULT_CHUNK_BYTES):
    """``filepath`` as a compact slab of ``shards`` N-range pieces over ``gpus`` devices (one piece on ``device`` when
    neither is given): a ``CompactSlab`` for one piece, a ``ShardedCompactSlab`` for more.

    * A ``CompactSlab.save`` file is copied piece by piece out of a memory map; ``K``, if given, must be the file's.
    * A dense (H, N, C) fp32 / fp16 / bf16 file is compacted at ``K`` on the devices as it streams in (one host thread
      per device, whole items per chunk of at most ``chunk_bytes``): no device holds more than its compact pieces plus
      one chunk.  Every piece has the bits of ``CompactSlab.from_dense`` of the whole slab (a 16-bit file: of its fp32
      widening).  ``slab.compaction`` then holds ``dropped_max`` (H,) fp32, the largest score dropped, and ``flat_rows``
      (H,) int64, the rows whose remainder reaches ``probs[0]`` (see ``CompactSlab.from_dense``)."""
    import concurrent.futures as cf
    obj = _open_compact(filepath)
    if obj is not None:
        H, N, Kf = (int(s) for s in obj["ids"].shape)
        C = int(obj["C"])
        if K is not None and int(K) != Kf:
            raise ValueError(f"{filepath}: a compact slab saved at K = {Kf}; K = {K} was asked for")
        K = Kf
    else:
        full = _open_mmap(filepath)
        H, N, C = (int(s) for s in full.shape)
        if full.dtype not in _KEPT_DTYPES:
            raise TypeError(f"{filepath}: compacting takes a float32, float16 or bfloat16 slab, got {full.dtype}")
        K = _check_k(K, C)
    dev = torch.device(device)
    home = dev.index if dev.index is not None else torch.cuda.current_device()
    plan = _load_plan(N, dev, shards, gpus)
    pieces, by_dev = [], {}
    for lo, hi, d in plan:
        dd = torch.device("cuda", d)
        p = CompactSlab(torch.empty((H, hi - lo, K), dtype=torch.int16, device=dd),
                        torch.empty((H, hi - lo, K), dtype=torch.float32, device=dd), C)
        pieces.append(p)
        by_dev.setdefault(d, []).append((p, lo, hi))
    with cf.ThreadPoolExecutor(max_workers=len(by_dev)) as ex:     # one host thread per device
        if obj is not None:
            futs = [ex.submit(_copy_compact_device, obj, todo) for todo in by_dev.values()]
        else:
            futs = [ex.submit(_compact_device, full, todo, K, chunk_bytes) for todo in by_dev.values()]
        outs = [f.result() for f in futs]
    compaction = None
    if obj is None:
        homedev = torch.device("cuda", home)
        flags = 0
        dropped = torch.zeros(H, dtype=torch.float32, device=homedev)
        flat = torch.zeros(H, dtype=torch.int64, device=homedev)
        for dm, fr, fl in outs:
            dropped = torch.maximum(dropped, dm.to(homedev))
            flat += fr.to(homedev)
            flags |= fl
        _raise_input_flags(flags)
        compaction = {"dropped_max": dropped, "flat_rows": flat}
    slab = pieces[0] if len(pieces) == 1 else ShardedCompactSlab(pieces)
    slab.compaction = compaction
    return slab


class Dataset:
    """(H, N, C) post-softmax scores from ``filepath`` (+ optional ``*_labels.pt``), forced to fp32
    (coda/datasets.py:12-23).  ``keep_dtype=True`` keeps a stored fp16 or bf16 slab at its width.

    With ``shards=`` / ``gpus=`` the slab is loaded as a ``ShardedSlab`` of N-range pieces over the GPUs
    (``load_sharded``) and never held whole on one device; ``chunk_bytes`` bounds its staging chunks.

    A file written by ``CompactSlab.save`` loads as a compact slab, and ``compact_k=K`` compacts a dense file at K as it
    loads (``load_compact``; a ``ShardedCompactSlab`` with more than one piece).

    ``host=True`` keeps the slab in host memory as a ``HostSlab`` over the file's memory map, computed on ``device``
    (``load_host``); with ``shards=`` / ``gpus=`` as well, as a ``ShardedHostSlab`` of N-range pieces of that memory
    map, each computed on its own device."""

    def __init__(self, filepath, device, keep_dtype=False, *, shards=None, gpus=None, chunk_bytes=DEFAULT_CHUNK_BYTES,
                 compact_k=None, host=False):
        self.device = device
        if compact_k or is_compact_file(filepath):
            self.preds = load_compact(filepath, device, compact_k, shards=shards, gpus=gpus, chunk_bytes=chunk_bytes)
        elif host:
            self.preds = load_host(filepath, device, keep_dtype, shards=shards, gpus=gpus)
        elif shards or gpus:
            self.preds = load_sharded(filepath, device, keep_dtype, shards=shards, gpus=gpus, chunk_bytes=chunk_bytes)
        else:
            preds = torch.load(filepath, map_location=device)
            self.preds = preds.to(_slab_dtype(preds, keep_dtype)).contiguous()
        print("Loaded preds of shape", self.preds.shape)
        self.labels = None
        label_p = filepath.replace(".pt", "_labels.pt")
        if os.path.exists(label_p):
            self.labels = torch.load(label_p, map_location=device)
            print("Loaded labels of shape", self.labels.shape)
        else:
            print("Did not load labels.")


class TensorDataset:
    """Wrap tensors already in memory.  ``n_offset``/``n_global`` describe an N-axis shard."""

    def __init__(self, preds, labels=None, n_offset=0, n_global=None):
        self.preds, self.labels, self.device = preds, labels, preds.device
        self.n_offset = n_offset
        self.n_global = preds.shape[1] if n_global is None else n_global


class ShardedFileDataset(TensorDataset):
    """This rank's contiguous N-range of an (H, N, C) ``.pt`` slab, read through ``torch.load(mmap=True)`` so that
    no rank ever materialises the whole tensor (the reference loader, coda/datasets.py:14, loads all of it onto
    one device).  Labels (``*_labels.pt``, N int64) are small and replicated.  ``keep_dtype``: see ``Dataset``."""

    def __init__(self, filepath, device, rank=0, world=1, keep_dtype=False):
        full = torch.load(filepath, map_location="cpu", mmap=True, weights_only=True)
        if full.dim() != 3:
            raise ValueError(f"{filepath}: expected an (H, N, C) tensor, got shape {tuple(full.shape)}")
        n = int(full.shape[1])
        lo, hi = shard_range(n, rank, world)
        if keep_dtype:
            preds = full[:, lo:hi].to(_slab_dtype(full, True)).contiguous().to(device)
        else:
            preds = full[:, lo:hi].float().contiguous().to(device)     # avoid fp16 precision errors (coda/datasets.py:14)
        labels = None
        label_p = filepath.replace(".pt", "_labels.pt")
        if os.path.exists(label_p):
            labels = torch.load(label_p, map_location="cpu", weights_only=True)
        super().__init__(preds, labels, n_offset=lo, n_global=n)
        self.labels_host = labels


class SyntheticDataset(TensorDataset):
    """This rank's shard of the synthetic task (SURVEY.md 8d); labels are replicated (N int64)."""

    def __init__(self, H, N, C, seed=0, device="cuda", dense=False, rank=0, world=1, generator_device=None,
                 dtype=torch.float32):
        lo, hi = shard_range(N, rank, world)
        gdev = generator_device or device
        preds, _ = synth(H, N, C, seed, device=gdev, dense=dense, n_lo=lo, n_hi=hi, dtype=dtype)
        _, labels = synth(H, N, C, seed, device=gdev, dense=dense, want_preds=False)
        super().__init__(preds.to(device), labels, n_offset=lo, n_global=N)
        self.labels_host = labels.cpu()


class CompactSlab:
    """Top-K + uniform-remainder form of an (H, N, C) score slab (``csrc/compact.cu``): ``ids`` (H, N, K) int16 holding
    uint16 class ids in descending score order, ``probs`` (H, N, K) float32; every other class of (h, n) gets
    ``(1 - sum_j probs) / (C - K)``.  24 bytes per (model, item) at K = 4 -- BASELINE.json configs[4] is 98 GB this way
    and 16.4 TB dense.  Duck-types the few tensor attributes the selector reads from ``dataset.preds``."""

    def __init__(self, ids: torch.Tensor, probs: torch.Tensor, C: int):
        if ids.shape != probs.shape or ids.dim() != 3 or ids.dtype != torch.int16 or probs.dtype != torch.float32:
            raise TypeError("CompactSlab: ids (H, N, K) int16 and probs (H, N, K) float32 expected")
        if ids.stride() != probs.stride() or ids.stride(2) != 1 or ids.stride(1) != ids.shape[2]:
            raise ValueError("CompactSlab: ids and probs must share strides, items contiguous")
        self.ids, self.probs, self.C = ids, probs, int(C)
        self.K = int(ids.shape[2])
        self.shape = (int(ids.shape[0]), int(ids.shape[1]), self.C)
        self.device = ids.device
        self.is_cuda = ids.is_cuda
        self.dtype = torch.float32
        self.compaction = None               # from_dense / load_compact: {"dropped_max", "flat_rows"} per model

    @classmethod
    def from_dense(cls, preds: torch.Tensor, K: int) -> "CompactSlab":
        """The top-K form of a CUDA (H, N, C) fp32 / fp16 / bf16 slab or N-range view of one, built on its device
        (``coda_b200_compact_build``): per (h, n) the K highest scores in descending order, equal scores by ascending
        class, so ``ids[..., 0]`` is ``torch.argmax``'s first-index maximum and ``probs`` the scores' exact fp32 bits.
        ``K`` in (1, 2, 3, 4, 8), K < C <= 4096.  Non-finite scores or scores outside [0, 1.0001] raise as a dense slab
        does.

        ``compaction`` holds two per-model diagnostics to choose K by: ``dropped_max`` (H,) fp32, the largest score the
        compaction drops (the max over items of the (K+1)-th score), and ``flat_rows`` (H,) int64, the items whose
        uniform remainder ``(1 - sum probs) * fp32(1 / (C - K))`` is >= ``probs[0]`` -- the only items where the arg-max
        of ``densify()`` can differ from ``ids[0]``."""
        from . import _native as nat
        if not (isinstance(preds, torch.Tensor) and preds.dim() == 3 and preds.is_cuda):
            raise TypeError("CompactSlab.from_dense: a CUDA (H, N, C) tensor expected")
        fmt = nat.slab_format(preds.dtype)
        H, N, C = (int(s) for s in preds.shape)
        K = _check_k(K, C)
        if not (preds.stride(2) == 1 and preds.stride(1) == C and (H == 1 or preds.stride(0) >= N * C)):
            raise ValueError("CompactSlab.from_dense: preds must be (H, N, C) with contiguous items")
        dev = preds.device
        ids = torch.empty((H, N, K), dtype=torch.int16, device=dev)
        probs = torch.empty((H, N, K), dtype=torch.float32, device=dev)
        dropped = torch.zeros(H, dtype=torch.float32, device=dev)
        flat = torch.zeros(H, dtype=torch.int64, device=dev)
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        if N:
            with torch.cuda.device(dev):
                _compact_launch(nat.load(), preds.data_ptr(), fmt, preds.stride(0) if H > 1 else N * C, H, N, C, K,
                                ids.data_ptr(), probs.data_ptr(), N * K, dropped.data_ptr(), flat.data_ptr(),
                                flags.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
        _raise_input_flags(int(flags.item()))
        slab = cls(ids, probs, C)
        slab.compaction = {"dropped_max": dropped, "flat_rows": flat}
        return slab

    def save(self, path):
        """Write this slab as a ``torch.save`` zip file ``{"format": "coda_b200.compact", "version": 1, "ids", "probs",
        "C"}``; ``load_compact`` (and the ``Dataset`` loaders) read it back, whole or as N-range pieces."""
        torch.save({"format": COMPACT_FORMAT, "version": COMPACT_VERSION, "ids": self.ids.contiguous().cpu(),
                    "probs": self.probs.contiguous().cpu(), "C": self.C}, path)

    def numel(self):
        return self.ids.numel() * 2          # what it costs relative to a dense float count (for the auto-shard rule)

    def narrow_items(self, lo, hi):
        return CompactSlab(self.ids[:, lo:hi], self.probs[:, lo:hi], self.C)

    def to(self, device):
        return CompactSlab(self.ids.to(device).contiguous(), self.probs.to(device).contiguous(), self.C)

    def densify(self) -> torch.Tensor:
        """The dense (H, N, C) float32 slab this form stands for (tests / small cases): same fp32 arithmetic for the
        remainder as the kernels (left-to-right sum of the K scores, 1 - s, times fp32(1 / (C - K)))."""
        H, N, C = self.shape
        s = self.probs[..., 0].clone()
        for j in range(1, self.K):
            s = s + self.probs[..., j]
        inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(C - self.K), dtype=torch.float32)
        rest = (1.0 - s) * inv.to(s.device)
        dense = rest[..., None].expand(H, N, C).clone()
        dense.scatter_(2, (self.ids.to(torch.int64) & 0xFFFF), self.probs)
        return dense

    def item_column(self, idx) -> torch.Tensor:
        """The dense (H, C) float32 scores of item ``idx``: bit-identical to ``densify()[:, idx]`` (the same
        element-wise fp32 operations), without densifying anything else."""
        H, _, C = self.shape
        p = self.probs[:, idx]
        s = p[:, 0].clone()
        for j in range(1, self.K):
            s = s + p[:, j]
        inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(C - self.K), dtype=torch.float32)
        rest = (1.0 - s) * inv.to(s.device)
        col = rest[:, None].expand(H, C).clone()
        col.scatter_(1, (self.ids[:, idx].to(torch.int64) & 0xFFFF), p)
        return col


class ShardedCompactSlab(PieceSlab):
    """A ``PieceSlab`` of ``CompactSlab`` pieces: the compact twin of ``ShardedSlab``.  CODA and the competing selectors
    give the bits of the whole ``CompactSlab`` with ``shards=`` the piece count."""

    def __init__(self, pieces):
        super().__init__(pieces)
        self.shape = tuple(self.shape)
        self.C, self.K = self.shape[2], self.pieces[0].K
        self.compaction = None

    @staticmethod
    def _check(pieces):
        for p in pieces:
            if not isinstance(p, CompactSlab):
                raise TypeError("ShardedCompactSlab: pieces must be CompactSlab (dense pieces make a ShardedSlab)")
            if p.shape[1] < 1:
                raise ValueError("ShardedCompactSlab: every piece must hold at least one item")
        H, _, C = pieces[0].shape
        K = pieces[0].K
        if any(p.shape[0] != H or p.C != C or p.K != K for p in pieces):
            raise TypeError("ShardedCompactSlab: all pieces must share H, C and K")

    def numel(self):
        return sum(p.numel() for p in self.pieces)


class CompactDataset:
    def __init__(self, slab: CompactSlab, labels=None, n_offset=0, n_global=None):
        self.preds, self.labels, self.device = slab, labels, slab.device
        self.n_offset = n_offset
        self.n_global = slab.shape[1] if n_global is None else n_global


class SyntheticCompactDataset(CompactDataset):
    """This rank's shard of the synthetic task generated directly in the compact form (the dense slab never exists)."""

    def __init__(self, H, N, C, K=4, seed=0, device="cuda", rank=0, world=1):
        lo, hi = shard_range(N, rank, world)
        ids, probs, _ = synth_compact(H, N, C, K, seed, device=device, n_lo=lo, n_hi=hi)
        _, _, labels = synth_compact(H, N, C, K, seed, device=device, want_slab=False)
        super().__init__(CompactSlab(ids, probs, C), labels, n_offset=lo, n_global=N)
        self.labels_host = labels.cpu()
