"""ModelPicker's unsupervised epsilon grid search on the GPU, and ``python -m coda_b200.eps_search``, its command line.

The search (the reference's ``scripts/modelselector/modelselector_eps_gridsearch_v2.py``, restated): draw ``iterations``
random pools ("realisations") of ``pool_size`` items, label each pool with the majority vote of the models, run
ModelPicker for ``budget`` steps per (epsilon, pool), and score each epsilon by how often its best model is one of the
pool's most accurate models.  Every run executes on the device in ``csrc/eps_search.cu`` (one launch covers all steps of
a wave of realisations times all epsilons); the metrics are computed on the host in float64.

The search reads the task only through its predicted classes (``hard_labels``: the [N][H] table of the selectors' slab
scan and a disagreement byte per item, as N-range pieces), so it runs on every slab layout -- one device tensor, a
compact slab, a host-resident slab, N-range pieces on several GPUs -- and the slab can be dropped before it starts.  The
realisations are split over one or more runner GPUs in contiguous blocks; per block, each piece copies the rows its
items hold into a pool table on the runner (``coda_b200_pool_gather``) and the runs read that table.

Run (e, r) is bit for bit ``ModelPicker(TensorDataset(preds[:, pool_r]), epsilon=epsilons[e]).run_steps(budget,
labels[pool_r], seed=eps_search_run_key(seed, e, r))``: its picks and best models equal ``history()[0]`` and
``best_history()[0]`` of that selector.

The best epsilons it writes (``best_epsilons.json``, ``{task: {"best_avg": ..., "best_fast": ...}}``) are what
``coda.baselines.modelpicker.TASK_EPS`` loads when ``CODA_B200_TASK_EPS`` names the file.
"""
from __future__ import annotations

import argparse
import json
import os

import numpy as np
import torch

from . import _native as nat

DEFAULT_EPSILONS = (0.35, 0.36, 0.37, 0.38, 0.39, 0.40, 0.41, 0.42, 0.43, 0.44, 0.45, 0.46, 0.47, 0.48, 0.49)
RESULTS_FILE = "best_epsilons.json"
_M64 = (1 << 64) - 1


def _splitmix64(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def eps_search_run_key(seed, e, r):
    """Philox key (an unsigned 64-bit int) of run (epsilon index ``e``, realisation ``r``) of a search made with
    ``seed``; ``ModelPicker.run_steps(..., seed=key)`` on that run's pool replays it."""
    return _splitmix64(_splitmix64(int(seed) & _M64) ^ _splitmix64(((int(e) & 0xFFFFFFFF) << 32) | (int(r) & 0xFFFFFFFF)))


def create_realisations(num_items, num_reals, pool_size):
    """``num_reals`` random pools of ``pool_size`` distinct items, from NumPy's global state (one permutation each)."""
    return np.array([np.random.permutation(num_items)[:pool_size] for _ in range(num_reals)])


def smooth(x, kernel_size=5):
    """Moving average with edge-value padding, as long as ``x``."""
    pad = kernel_size // 2
    xp = np.concatenate([np.full(pad, x[0]), x, np.full(pad, x[-1])])
    return np.convolve(xp, np.ones(kernel_size) / kernel_size, "valid")


def search_metrics(best, pool_accuracies, pool_size, epsilons, threshold):
    """The search's scores from the best model of every step, ``best`` [E][R][B], and the integer pool accuracies
    [R][H].  Per epsilon: ``success_mean`` [B] (the share of realisations whose best model is among the pool's exact
    arg-max models), ``acc_mean`` [B] (the mean pool accuracy of the best model), ``avg_success`` (the mean of
    success_mean) and ``fastest_t`` (the first step where success_mean reaches ``threshold``, ``inf`` when the smoothed
    curve is not above it there).  -> (best_avg, best_fast, metrics): the first epsilon of highest avg_success and of
    lowest fastest_t."""
    acc = np.asarray(pool_accuracies, dtype=np.int64)
    frac = acc / pool_size
    top = acc.max(axis=1, keepdims=True)
    rows = np.arange(acc.shape[0])[:, None]
    metrics = {}
    for e, eps in enumerate(epsilons):
        b = np.asarray(best[e], dtype=np.int64)
        success = np.ascontiguousarray((acc[rows, b] == top).astype(np.int64))
        success_mean = np.mean(success, axis=0)
        acc_mean = np.mean(np.ascontiguousarray(frac[rows, b]), axis=0)
        t = int(np.argmax(success_mean >= threshold))
        fastest = t if smooth(success_mean)[t] > threshold else float("inf")
        metrics[float(eps)] = {"success_mean": success_mean.tolist(), "acc_mean": acc_mean.tolist(),
                               "avg_success": float(np.mean(success_mean)), "fastest_t": fastest}
    best_avg = max(metrics.items(), key=lambda kv: kv[1]["avg_success"])[0]
    best_fast = min(metrics.items(), key=lambda kv: kv[1]["fastest_t"])[0]
    return best_avg, best_fast, metrics


def _check_epsilons(epsilons):
    eps = [float(e) for e in epsilons]
    if not eps:
        raise ValueError("modelpicker_eps_search: no epsilons given")
    for e in eps:
        if not 0.0 < e < 1.0:
            raise ValueError(f"modelpicker_eps_search: epsilon must be in (0, 1), got {e}")
    return eps


POOL_TABLE_BYTES = 1 << 30      # device bytes of one block's pool table: rows, disagreement bytes and labels


class HardLabels:
    """What ModelPicker's search reads of a task: every model's predicted class of every item, as N-range pieces.
    ``pieces`` = [(hard [N_i][H] (uint16 class ids as int16), disagree [N_i] uint8, n_offset)], each on the device whose
    slab scan made it; ``shape`` = (H, N, C).  Built by ``hard_labels``; it holds no reference to the slab, so the
    slab can be dropped once it exists.  [N][H] at 2 bytes per model and item: 512 MB at H = 256, N = 1e6."""

    def __init__(self, pieces, shape):
        self.pieces = list(pieces)
        self.shape = tuple(int(s) for s in shape)

    @property
    def devices(self):
        """The indices of the devices the pieces are on, ascending."""
        return sorted({h.device.index for h, _, _ in self.pieces})


def _whole_task(dataset, preds):
    """(H, N, C) of a slab the search takes: the whole task, at most 1024 models, in one process."""
    from .dist import default_comm
    if preds is None or len(preds.shape) != 3:
        raise TypeError("modelpicker_eps_search: dataset.preds must be an (H, N, C) slab")
    H, N, C = (int(s) for s in preds.shape)
    if H > 1024:
        raise NotImplementedError("coda_b200: H > 1024 models is not supported yet")
    if int(getattr(dataset, "n_global", N)) != N or default_comm().world > 1:
        raise NotImplementedError("modelpicker_eps_search: runs over the whole task in one process; an N-range shard "
                                  "of it (one process per GPU) is not supported")
    return H, N, C


def hard_labels(dataset):
    """The ``HardLabels`` of ``dataset.preds``, one piece per piece of the slab, each made by the slab scan the
    selectors run (``_DeviceState.scan``) on the piece's device: a dense fp32 / fp16 / bf16 tensor or a ``CompactSlab``
    (one piece), a ``HostSlab`` (one piece, streamed through its device in chunks), or the pieces of a ``ShardedSlab``,
    ``ShardedCompactSlab`` or ``ShardedHostSlab`` (one host thread per device).  Non-finite or out-of-range scores
    raise as the selectors raise them."""
    import concurrent.futures as cf
    from .baselines import _DeviceState
    from .datasets import pieces_of
    preds = getattr(dataset, "preds", None)
    shape = _whole_task(dataset, preds)
    states = [_DeviceState(p, off) for p, off in pieces_of(preds)]

    def scan(sts):
        out = []
        for st in sts:
            hard, disagree, _ = st.scan(ens=False)
            out.append((hard, disagree, st.n_offset))
            st.close()
        return out

    by_dev = {}
    for st in states:
        by_dev.setdefault(st.dev, []).append(st)
    with cf.ThreadPoolExecutor(max_workers=len(by_dev)) as ex:
        done = [f.result() for f in [ex.submit(scan, sts) for sts in by_dev.values()]]
    pieces = sorted((p for ps in done for p in ps), key=lambda p: p[2])
    return HardLabels(pieces, shape)


def realisation_blocks(R, runners, per_block):
    """[[(r0, r1)] of each runner]: runner j takes the contiguous realisations ``shard_range(R, j, runners)``, in
    blocks of at most ``per_block`` realisations, in order."""
    from .synth import shard_range
    out = []
    for j in range(runners):
        lo, hi = shard_range(R, j, runners)
        out.append([(a, min(hi, a + per_block)) for a in range(lo, hi, per_block)])
    return out


def pool_table(pools, offsets):
    """The pool table of the realisations ``pools`` [R_b, P] (global item ids) over pieces starting at items
    ``offsets`` (ascending, the first 0): the rows of the pool positions in pool-major order, grouped by piece, so that
    the table is the concatenation of what each piece gathers.  -> (local [R_b, P], the row of each pool position in
    that table; [items of piece i, local to it, in pool-major order])."""
    flat = np.ascontiguousarray(pools, dtype=np.int64).reshape(-1)
    offsets = np.asarray(offsets, dtype=np.int64)
    piece = (np.searchsorted(offsets, flat, side="right") - 1).astype(np.int16)   # int16: a stable sort is a radix sort
    order = np.argsort(piece, kind="stable")
    local = np.empty_like(flat)
    local[order] = np.arange(flat.size, dtype=np.int64)
    counts = np.bincount(piece, minlength=offsets.size)
    items = np.split(flat[order] - offsets[piece[order]], np.cumsum(counts)[:-1])
    return local.reshape(np.shape(pools)), items


def _gather(lib, hard, disagree, labels, slots, items, out_hard, out_disagree, out_labels):
    """``coda_b200_pool_gather`` of one piece on its device's current stream."""
    from .baselines import _ptr
    H = int(hard.shape[1])
    nat.check(lib.coda_b200_pool_gather(_ptr(hard), _ptr(disagree), _ptr(labels), H, _ptr(slots), _ptr(items),
                                        int(items.numel()), _ptr(out_hard), _ptr(out_disagree), _ptr(out_labels),
                                        torch.cuda.current_stream(hard.device).cuda_stream), "pool_gather")


def _stage_block(lib, table, labs, pools, dev, gammas, keys, B):
    """First phase of one block on runner ``dev``: upload its indices, gather the pool table of realisations ``pools``
    [R_b, P] from every piece (``keys`` [E][R_b]) and allocate its outputs.  Nothing here waits for a run: the index
    uploads are the only host-blocking copies, and they come before any runner's runs are enqueued.  -> the block's
    device arrays by name."""
    H = table.shape[0]
    R, P = pools.shape
    E = len(gammas)
    local, items = pool_table(pools, [off for _, _, off in table.pieces])
    with torch.cuda.device(dev):
        b = {"hard": torch.empty((R * P, H), dtype=torch.int16, device=dev),
             "disagree": torch.empty(R * P, dtype=torch.uint8, device=dev),
             "labels": torch.empty(R * P, dtype=torch.int64, device=dev)}
        base = 0
        for (hard, dis, _), lab, it in zip(table.pieces, labs, items):
            k, pd = int(it.size), hard.device
            if k == 0:
                continue
            with torch.cuda.device(pd):
                it_d = torch.from_numpy(it).to(pd)
                if pd == dev:                                  # straight into the runner's table
                    _gather(lib, hard, dis, lab, torch.arange(base, base + k, device=pd), it_d, b["hard"],
                            b["disagree"], b["labels"])
                else:                                          # a compact output, then one copy per array
                    bh = torch.empty((k, H), dtype=torch.int16, device=pd)
                    bd = torch.empty(k, dtype=torch.uint8, device=pd)
                    bl = torch.empty(k, dtype=torch.int64, device=pd)
                    _gather(lib, hard, dis, lab, torch.arange(k, device=pd), it_d, bh, bd, bl)
            if pd != dev:
                b["hard"][base:base + k].copy_(bh)
                b["disagree"][base:base + k].copy_(bd)
                b["labels"][base:base + k].copy_(bl)
            base += k
        b["pool"] = torch.from_numpy(local).to(dev)
        b["gammas"] = torch.from_numpy(gammas).to(dev)
        b["keys"] = torch.from_numpy(np.ascontiguousarray(keys).view(np.int64)).to(dev)
        b["acc"] = torch.empty((R, H), dtype=torch.int32, device=dev)
        for name, dt in (("picks", torch.int32), ("best", torch.int32), ("pick_tie", torch.uint8),
                         ("best_tie", torch.uint8)):
            b[name] = torch.empty((E, R, B), dtype=dt, device=dev)
        b["flags"] = torch.zeros(1, dtype=torch.int32, device=dev)
    b["dev"], b["R"], b["P"] = dev, R, P
    return b


def _launch_block(lib, b, H, C, B, E):
    """Second phase of one block: enqueue its pool accuracies and every step of its runs on the runner's current
    stream (launches only; nothing waits)."""
    from .baselines import _ptr
    dev, R, P = b["dev"], b["R"], b["P"]
    with torch.cuda.device(dev):
        s = torch.cuda.current_stream(dev).cuda_stream
        plan = np.zeros(5, dtype=np.int64)
        nat.check(lib.coda_b200_mp_runs_plan(H, E, P, R, B, plan.ctypes.data), "mp_runs_plan")
        b["scratch"] = torch.empty(max(int(plan[4]), 1), dtype=torch.uint8, device=dev)
        nat.check(lib.coda_b200_pool_accuracy(_ptr(b["hard"]), _ptr(b["labels"]), H, _ptr(b["pool"]), R, P,
                                              _ptr(b["acc"]), s), "pool_accuracy")
        nat.check(lib.coda_b200_mp_runs(_ptr(b["hard"]), _ptr(b["labels"]), _ptr(b["disagree"]), H, C, _ptr(b["pool"]),
                                        R, P, B, _ptr(b["gammas"]), _ptr(b["keys"]), E, _ptr(b["scratch"]),
                                        b["scratch"].numel(), _ptr(b["picks"]), _ptr(b["best"]), _ptr(b["pick_tie"]),
                                        _ptr(b["best_tie"]), _ptr(b["flags"]), s), "mp_runs")


def _enqueue_round(lib, table, labs, work, gammas, B):
    """One block on each runner, ``work`` = [(device, pools [R_b, P], keys [E][R_b])]: every block is staged (its
    gathers and copies enqueued, on the pieces' devices too) before any block's runs are launched, so no runner's
    gathers queue behind another runner's runs and the host never waits for a run while it enqueues.  -> the blocks'
    device arrays, in ``work`` order."""
    staged = [_stage_block(lib, table, labs, pools, dev, gammas, keys, B) for dev, pools, keys in work]
    for b in staged:
        _launch_block(lib, b, table.shape[0], table.shape[2], B, len(gammas))
    return staged


def _piece_labels(lib, table, labels):
    """Each piece's labels on its device: ``labels`` [N] (CPU int) sliced, or the majority vote, which is item-local."""
    from .baselines import _ptr
    H = table.shape[0]
    labs = []
    for hard, _, off in table.pieces:
        n, pd = int(hard.shape[0]), hard.device
        with torch.cuda.device(pd):
            if labels is None:
                lab = torch.empty(n, dtype=torch.int64, device=pd)
                nat.check(lib.coda_b200_majority(_ptr(hard), H, n, _ptr(lab), torch.cuda.current_stream(pd).cuda_stream),
                          "majority")
            else:
                lab = labels[off:off + n].to(device=pd, dtype=torch.int64)
        labs.append(lab)
    return labs


def _table_budget(runners):
    """Device bytes one block's pool table may take: ``POOL_TABLE_BYTES``, but at most a quarter of the memory the
    runner with the least of it has free (torch's cached, unused blocks counted as free)."""
    free = min(torch.cuda.mem_get_info(d)[0] + torch.cuda.memory_reserved(d) - torch.cuda.memory_allocated(d)
               for d in runners)
    return min(POOL_TABLE_BYTES, free // 4)


def _search_table(table, pools, gammas, keys, B, labels, runners):
    """Every run of the search on ``table`` (``HardLabels``), its realisations split over the ``runners`` (device
    indices) in blocks whose pool table fits ``_table_budget``.  Each round stages one block on every runner, then
    launches them all, then reads them back.  -> (host outputs by name, the OR of the runners' flags words)."""
    lib = nat.load()
    H, N, C = table.shape
    R, P = pools.shape
    E = len(gammas)
    labs = _piece_labels(lib, table, labels)
    per_block = max(1, _table_budget(runners) // (P * (2 * H + 1 + 8)))
    blocks = realisation_blocks(R, len(runners), per_block)
    out = {"picks": np.empty((E, R, B), np.int32), "best": np.empty((E, R, B), np.int32),
           "pick_tie": np.empty((E, R, B), np.uint8), "best_tie": np.empty((E, R, B), np.uint8),
           "pool_accuracies": np.empty((R, H), np.int32)}
    flags = 0
    for rnd in range(max(len(b) for b in blocks)):
        spans = [(d, b[rnd]) for d, b in zip(runners, blocks) if rnd < len(b)]
        staged = _enqueue_round(lib, table, labs, [(torch.device("cuda", d), pools[r0:r1], keys[:, r0:r1])
                                                   for d, (r0, r1) in spans], gammas, B)
        for (_, (r0, r1)), b in zip(spans, staged):
            for name in ("picks", "best", "pick_tie", "best_tie"):
                out[name][:, r0:r1] = b[name].cpu().numpy()
            out["pool_accuracies"][r0:r1] = b["acc"].cpu().numpy()
            flags |= int(b["flags"].item())
        del staged
    out["labels"] = torch.cat([lab.cpu() for lab in labs]).numpy()
    return out, flags


def modelpicker_eps_search(dataset, epsilons=DEFAULT_EPSILONS, iterations=1000, pool_size=1000, budget=1000,
                           threshold=0.9, *, seed=None, realisations=None, labels=None, gpus=None):
    """ModelPicker's epsilon grid search on ``dataset`` (the whole task), or on its ``HardLabels``.

    ``dataset``: a dataset whose ``preds`` is one device tensor or a whole ``CompactSlab`` (its ``hard_labels`` are
    built, searched and dropped), or the ``HardLabels`` of any slab layout (``hard_labels(dataset)``: N-range pieces,
    host-resident slabs).  ``gpus``: the realisations run on ``cuda:0`` .. ``cuda:gpus-1``, a contiguous block each
    (default: the devices the table's pieces are on); the runs never talk to each other, so every run's bits are the
    same for any layout and any ``gpus``.  Each runner holds one block's pool table at a time: up to 1 GiB
    (``POOL_TABLE_BYTES``) and at most a quarter of its free memory.

    ``realisations``: an [R, P] array of item indices; by default ``iterations`` pools drawn with
    ``np.random.permutation(N)[:pool_size]`` each from NumPy's global state.  ``pool_size`` is clamped to N and
    ``budget`` to the pool size.  ``labels``: the oracle, N class ids; by default the majority vote of the models (the
    smallest class among equal counts).  ``seed``: the search's Philox seed (``None``: one ``torch.randint`` on the CPU
    generator); run (e, r) uses ``eps_search_run_key(seed, e, r)``.

    Returns a dict: ``best_avg``, ``best_fast``, ``metrics`` (per epsilon, see ``search_metrics``), and the raw
    ``picks`` / ``best`` / ``pick_tie`` / ``best_tie`` [E, R, B] arrays (pool positions and models of every step),
    ``realisations`` [R, P], ``pool_accuracies`` [R, H], ``labels`` [N], ``epsilons``, ``seed``."""
    eps = _check_epsilons(epsilons)
    from .datasets import HostSlab, PieceSlab
    if isinstance(dataset, HardLabels):
        H, N, C = dataset.shape
    else:
        preds = getattr(dataset, "preds", None)
        if isinstance(preds, (PieceSlab, HostSlab)):
            raise NotImplementedError(f"modelpicker_eps_search: a {type(preds).__name__} (a slab loaded as N-range "
                                      f"pieces or kept in host memory) is searched through its predicted-class table: "
                                      f"modelpicker_eps_search(coda_b200.eps_search.hard_labels(dataset), ...)")
        H, N, C = _whole_task(dataset, preds)
    if gpus is not None and not 1 <= int(gpus) <= torch.cuda.device_count():
        raise ValueError(f"modelpicker_eps_search: gpus={gpus}, but {torch.cuda.device_count()} GPUs are visible")
    if realisations is None:
        if int(iterations) < 1 or int(pool_size) < 1:
            raise ValueError("modelpicker_eps_search: iterations and pool_size must be >= 1")
        pools = create_realisations(N, int(iterations), min(int(pool_size), N))
    else:
        pools = np.asarray(realisations)
        if pools.ndim != 2 or pools.shape[0] < 1 or pools.shape[1] < 1 or not np.issubdtype(pools.dtype, np.integer):
            raise ValueError("modelpicker_eps_search: realisations must be a non-empty [R, P] array of item indices")
        if pools.min() < 0 or pools.max() >= N:
            raise ValueError(f"modelpicker_eps_search: realisations hold items outside [0, {N})")
    R, P = (int(s) for s in pools.shape)
    B = min(int(budget), P)
    if B < 1:
        raise ValueError("modelpicker_eps_search: budget must be >= 1")
    if labels is not None:
        lab = torch.as_tensor(np.asarray(labels.cpu() if isinstance(labels, torch.Tensor) else labels))
        if lab.dim() != 1 or lab.numel() != N or lab.is_floating_point():
            raise ValueError(f"modelpicker_eps_search: labels must be {N} integer class ids")
    if seed is None:
        seed = int(torch.randint(0, 1 << 62, (1,)).item())
    E = len(eps)
    gammas = np.array([np.float32((1.0 - e) / e) for e in eps], dtype=np.float32)   # ModelPicker's fp32 gamma
    keys = np.array([[eps_search_run_key(seed, e, r) for r in range(R)] for e in range(E)], dtype=np.uint64)
    table = dataset if isinstance(dataset, HardLabels) else hard_labels(dataset)
    runners = list(range(int(gpus))) if gpus is not None else table.devices
    out, flags = _search_table(table, np.ascontiguousarray(pools, dtype=np.int64), gammas, keys, B,
                               None if labels is None else lab, runners)
    del table
    if flags:
        raise RuntimeError("modelpicker_eps_search: a run found no item to label (non-finite entropies)")
    best_avg, best_fast, metrics = search_metrics(out["best"], out["pool_accuracies"], P, eps, threshold)
    return {"best_avg": best_avg, "best_fast": best_fast, "metrics": metrics, "realisations": pools,
            "epsilons": eps, "seed": int(seed), **out}


# -- command line -------------------------------------------------------------------------------------------------
def _parser():
    p = argparse.ArgumentParser(prog="python -m coda_b200.eps_search",
                                description="ModelPicker's unsupervised epsilon grid search on the GPU")
    p.add_argument("--preds", help="path to an (H, N, C) tensor of model predictions")
    p.add_argument("--pred-dir", default="data", help="directory of prediction tensors (.pt)")
    p.add_argument("--task", default=None, help="task name: <pred-dir>/<task>.pt")
    p.add_argument("--epsilons", default=",".join(f"{e:.2f}" for e in DEFAULT_EPSILONS))
    p.add_argument("--iterations", type=int, default=1000, help="number of random realisations")
    p.add_argument("--pool-size", type=int, default=1000, help="realisation pool size")
    p.add_argument("--budget", type=int, default=1000, help="labels per realisation")
    p.add_argument("--threshold", type=float, default=0.9, help="success threshold of the fastest metric")
    p.add_argument("--seed", type=int, default=None, help="seeds NumPy (the realisations) and the Philox keys")
    p.add_argument("--gpus", type=int, default=None,
                   help="keep the task in host memory, scan it on this many GPUs (one N-range piece each) and run "
                        "the realisations over them; also taken, with one GPU, when the task exceeds its free memory")
    return p


def _load_results(path):
    if os.path.exists(path):
        with open(path) as f:
            return json.load(f)
    return {}


def _auto_pieces(path, dev):
    """How the command line loads ``path`` without ``--gpus``: None for the plain load (``Dataset(path, dev)``), else
    the piece count of the table route.  A dense file whose fp32 slab exceeds the free memory of CUDA device ``dev``
    takes one host-resident piece on ``dev``.  A ``CompactSlab.save`` file that exceeds it takes one compact piece per
    visible GPU when there is more than one (a compact slab has no host-resident form, so with one GPU the plain load
    stands and fails as it would).  A file in torch's legacy format keeps the plain load."""
    from .datasets import _free_bytes, _open_compact, _open_mmap
    if dev.type != "cuda":
        return None
    obj = _open_compact(path)
    if obj is None:
        try:
            held = _open_mmap(path).numel() * 4
        except ValueError:                                         # legacy format: no memory map, keep the plain load
            return None
    else:
        held = obj["ids"].numel() * 6
    if held <= _free_bytes(dev.index if dev.index is not None else torch.cuda.current_device()):
        return None
    if obj is None:
        return 1
    return torch.cuda.device_count() if torch.cuda.device_count() > 1 else None


def _table_from_file(path, dev, gpus):
    """The ``HardLabels`` of ``path``, loaded as a host-resident slab over its memory map (``gpus`` > 1: that many
    N-range pieces, one per GPU) and dropped once scanned; a ``CompactSlab.save`` file loads onto the devices as compact
    pieces (one ``CompactSlab`` for ``gpus`` = 1)."""
    from .datasets import Dataset
    k = int(gpus or 1)
    if not 1 <= k <= torch.cuda.device_count():
        raise ValueError(f"--gpus {gpus}: {torch.cuda.device_count()} GPUs are visible")
    data = Dataset(path, dev, host=True, shards=k if k > 1 else None)
    table = hard_labels(data)
    del data
    return table


def _search_file(path, args, search):
    from .datasets import Dataset
    dev = torch.device("cuda" if torch.cuda.is_available() else "cpu")
    kw = dict(epsilons=[float(e) for e in args.epsilons.split(",")], iterations=args.iterations,
              pool_size=args.pool_size, budget=args.budget, threshold=args.threshold, seed=args.seed)
    pieces = args.gpus if args.gpus is not None else _auto_pieces(path, dev)
    if args.gpus is not None:
        kw["gpus"] = args.gpus
    data = Dataset(path, dev) if pieces is None else _table_from_file(path, dev, pieces)
    res = search(data, **kw)
    for eps, m in res["metrics"].items():
        print(f"eps={eps:.3f} avg_success={m['avg_success']:.3f} fastest_t={m['fastest_t']}")
    print("\nOptimal epsilon (avg_success):", res["best_avg"])
    print("Optimal epsilon (fastest):", res["best_fast"])
    return res


def main(argv=None, search=modelpicker_eps_search):
    """The command line: searches ``--task`` / ``--preds`` (or every ``.pt`` of ``--pred-dir`` but ``*_labels.pt``)
    and adds ``{key: {"best_avg", "best_fast"}}`` to ``best_epsilons.json`` in the working directory, skipping keys
    already there (key: the task name, else the file name).  ``search`` is the search function (a stand-in in tests)."""
    p = _parser()
    args = p.parse_args(argv)
    _check_epsilons(args.epsilons.split(","))
    if args.seed is not None:
        np.random.seed(args.seed)
    if args.task:
        args.preds = os.path.join(args.pred_dir, args.task + ".pt")
    if args.preds:
        todo = [(args.task or os.path.basename(args.preds), args.preds)]
    elif args.pred_dir:
        names = sorted(f for f in os.listdir(args.pred_dir) if f.endswith(".pt") and not f.endswith("_labels.pt"))
        todo = [(f, os.path.join(args.pred_dir, f)) for f in names]
    else:
        p.error("Either --preds, --pred-dir or --task must be specified")
    for key, path in todo:
        if key in _load_results(RESULTS_FILE):
            print(key, "already computed; skipping")
            continue
        res = _search_file(path, args, search)
        overall = _load_results(RESULTS_FILE)              # another process may have written meanwhile
        overall[key] = {"best_avg": res["best_avg"], "best_fast": res["best_fast"]}
        with open(RESULTS_FILE, "w") as f:
            json.dump(overall, f, indent=2)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
