"""ModelPicker's unsupervised epsilon grid search on the GPU, and ``python -m coda_b200.eps_search``, its command line.

The search (the reference's ``scripts/modelselector/modelselector_eps_gridsearch_v2.py``, restated): draw ``iterations``
random pools ("realisations") of ``pool_size`` items, label each pool with the majority vote of the models, run
ModelPicker for ``budget`` steps per (epsilon, pool), and score each epsilon by how often its best model is one of the
pool's most accurate models.  Every run executes on the device in ``csrc/eps_search.cu`` (one launch covers all steps of
a wave of realisations times all epsilons); the metrics are computed on the host in float64.

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


def modelpicker_eps_search(dataset, epsilons=DEFAULT_EPSILONS, iterations=1000, pool_size=1000, budget=1000,
                           threshold=0.9, *, seed=None, realisations=None, labels=None):
    """ModelPicker's epsilon grid search on ``dataset`` (the whole task, on one GPU).

    ``realisations``: an [R, P] array of item indices; by default ``iterations`` pools drawn with
    ``np.random.permutation(N)[:pool_size]`` each from NumPy's global state.  ``pool_size`` is clamped to N and
    ``budget`` to the pool size.  ``labels``: the oracle, N class ids; by default the majority vote of the models (the
    smallest class among equal counts).  ``seed``: the search's Philox seed (``None``: one ``torch.randint`` on the CPU
    generator); run (e, r) uses ``eps_search_run_key(seed, e, r)``.

    Returns a dict: ``best_avg``, ``best_fast``, ``metrics`` (per epsilon, see ``search_metrics``), and the raw
    ``picks`` / ``best`` / ``pick_tie`` / ``best_tie`` [E, R, B] arrays (pool positions and models of every step),
    ``realisations`` [R, P], ``pool_accuracies`` [R, H], ``labels`` [N], ``epsilons``, ``seed``."""
    from .baselines import _DeviceState, _ptr
    from .dist import default_comm
    eps = _check_epsilons(epsilons)
    from .datasets import HostSlab, ShardedCompactSlab, ShardedHostSlab, ShardedSlab
    preds = getattr(dataset, "preds", None)
    if isinstance(preds, (ShardedSlab, ShardedCompactSlab, HostSlab, ShardedHostSlab)):
        raise NotImplementedError(f"modelpicker_eps_search: runs on one GPU over one (H, N, C) tensor; a "
                                  f"{type(preds).__name__} (a slab loaded as N-range pieces or kept in host memory) is "
                                  f"not supported -- load the task as one device tensor")
    if preds is None or len(preds.shape) != 3:
        raise TypeError("modelpicker_eps_search: dataset.preds must be an (H, N, C) slab")
    H, N, C = (int(s) for s in preds.shape)
    if H > 1024:
        raise NotImplementedError("coda_b200: H > 1024 models is not supported yet")
    if int(getattr(dataset, "n_global", N)) != N or default_comm().world > 1:
        raise NotImplementedError("modelpicker_eps_search: runs on one GPU over the whole task; an N-range shard of it "
                                  "(one process per GPU) is not supported")
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

    st = _DeviceState(preds)
    lib, dev = st.lib, st.dev
    plan = np.zeros(5, dtype=np.int64)
    with st._on():
        nat.check(lib.coda_b200_mp_runs_plan(H, E, P, R, B, plan.ctypes.data), "mp_runs_plan")
        hard, disagree, _ = st.scan(ens=False)
        if labels is None:
            lab_d = torch.empty(N, dtype=torch.int64, device=dev)
            st._call("coda_b200_majority", _ptr(hard), H, N, _ptr(lab_d), st._s())
        else:
            lab_d = lab.to(device=dev, dtype=torch.int64).contiguous()
        pool_d = torch.from_numpy(np.ascontiguousarray(pools, dtype=np.int64)).to(dev)
        acc_d = torch.empty((R, H), dtype=torch.int32, device=dev)
        st._call("coda_b200_pool_accuracy", _ptr(hard), _ptr(lab_d), H, _ptr(pool_d), R, P, _ptr(acc_d), st._s())
        gam_d = torch.from_numpy(gammas).to(dev)
        keys_d = torch.from_numpy(keys.view(np.int64)).to(dev)
        scratch = torch.empty(max(int(plan[4]), 1), dtype=torch.uint8, device=dev)
        picks = torch.empty((E, R, B), dtype=torch.int32, device=dev)
        best = torch.empty((E, R, B), dtype=torch.int32, device=dev)
        ptie = torch.empty((E, R, B), dtype=torch.uint8, device=dev)
        btie = torch.empty((E, R, B), dtype=torch.uint8, device=dev)
        st.flags.zero_()
        st._call("coda_b200_mp_runs", _ptr(hard), _ptr(lab_d), _ptr(disagree), H, C, _ptr(pool_d), R, P, B,
                 _ptr(gam_d), _ptr(keys_d), E, _ptr(scratch), scratch.numel(), _ptr(picks), _ptr(best), _ptr(ptie),
                 _ptr(btie), _ptr(st.flags), st._s())
        flags = int(st.flags.item())
        out = {k: v.cpu().numpy() for k, v in (("picks", picks), ("best", best), ("pick_tie", ptie),
                                               ("best_tie", btie), ("pool_accuracies", acc_d), ("labels", lab_d))}
    del scratch, hard, disagree
    st.close()
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
    return p


def _load_results(path):
    if os.path.exists(path):
        with open(path) as f:
            return json.load(f)
    return {}


def _search_file(path, args, search):
    from .datasets import Dataset
    dev = torch.device("cuda" if torch.cuda.is_available() else "cpu")
    data = Dataset(path, dev)
    res = search(data, epsilons=[float(e) for e in args.epsilons.split(",")], iterations=args.iterations,
                 pool_size=args.pool_size, budget=args.budget, threshold=args.threshold, seed=args.seed)
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
