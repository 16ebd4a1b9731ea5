"""The epsilon grid search through its pool table (coda_b200.eps_search: hard_labels, coda_b200_pool_gather) against
the global-index launch it replaced, on one GPU, and the table path over several runner GPUs.

    python tools/bench_eps_search_table.py [--realisations 1000] [--pool-size 1000] [--budget 1000] [--reps 2]

The default grid is the reference script's (15 epsilons x 1000 realisations x pool 1000 x budget 1000) at H = 64 / C = 10
and H = 256 / C = 100, N = 20000 synthetic items.  "global" is the search before the pool table: coda_b200_majority,
coda_b200_pool_accuracy and coda_b200_mp_runs on the whole [N][H] table with global item ids, then the host metrics;
"table" is ``modelpicker_eps_search`` on the same ``HardLabels``.  Both start from the same scan, are timed alternately
in the same process (host clock around the call, device synchronised), and their outputs are compared bit for bit.
Then the table path with ``gpus`` = 1, 2, 4, 8 (as many as are visible), and the time ``hard_labels`` takes on a
host-resident file (``Dataset(path, host=True)``, written to a temporary directory).  Prints the card and its power
limit with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

EPS = (0.35, 0.36, 0.37, 0.38, 0.39, 0.40, 0.41, 0.42, 0.43, 0.44, 0.45, 0.46, 0.47, 0.48, 0.49)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def global_search(table, pools, seed, B):
    """The search's launches on global item ids over the whole table (one piece, on cuda:0)."""
    from coda_b200 import _native as nat
    from coda_b200.eps_search import eps_search_run_key, search_metrics
    lib = nat.load()
    (hard, dis, _), = table.pieces
    H, N, C = table.shape
    R, P = pools.shape
    E = len(EPS)
    dev = hard.device
    s = torch.cuda.current_stream(dev).cuda_stream
    gammas = np.array([np.float32((1.0 - e) / e) for e in EPS], dtype=np.float32)
    keys = np.array([[eps_search_run_key(seed, e, r) for r in range(R)] for e in range(E)], dtype=np.uint64)
    plan = np.zeros(5, dtype=np.int64)
    nat.check(lib.coda_b200_mp_runs_plan(H, E, P, R, B, plan.ctypes.data))
    lab = torch.empty(N, dtype=torch.int64, device=dev)
    nat.check(lib.coda_b200_majority(hard.data_ptr(), H, N, lab.data_ptr(), s))
    pool = torch.from_numpy(np.ascontiguousarray(pools, dtype=np.int64)).to(dev)
    acc = torch.empty((R, H), dtype=torch.int32, device=dev)
    nat.check(lib.coda_b200_pool_accuracy(hard.data_ptr(), lab.data_ptr(), H, pool.data_ptr(), R, P, acc.data_ptr(), s))
    gam = torch.from_numpy(gammas).to(dev)
    kd = torch.from_numpy(keys.view(np.int64)).to(dev)
    scratch = torch.empty(max(int(plan[4]), 1), dtype=torch.uint8, device=dev)
    out = [torch.empty((E, R, B), dtype=dt, device=dev) for dt in (torch.int32, torch.int32, torch.uint8, torch.uint8)]
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    nat.check(lib.coda_b200_mp_runs(hard.data_ptr(), lab.data_ptr(), dis.data_ptr(), H, C, pool.data_ptr(), R, P, B,
                                    gam.data_ptr(), kd.data_ptr(), E, scratch.data_ptr(), scratch.numel(),
                                    *[t.data_ptr() for t in out], flags.data_ptr(), s))
    assert int(flags.item()) == 0
    res = dict(zip(("picks", "best", "pick_tie", "best_tie", "pool_accuracies", "labels"),
                   [t.cpu().numpy() for t in out + [acc, lab]]))
    res["best_avg"], res["best_fast"], _ = search_metrics(res["best"], res["pool_accuracies"], P, EPS, 0.9)
    return res


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    for d in range(torch.cuda.device_count()):
        torch.cuda.synchronize(d)
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--realisations", type=int, default=1000)
    ap.add_argument("--pool-size", type=int, default=1000)
    ap.add_argument("--budget", type=int, default=1000)
    ap.add_argument("--items", type=int, default=20000, help="N of the synthetic task")
    ap.add_argument("--shapes", default="64x10,256x100", help="H x C of the synthetic tasks")
    ap.add_argument("--reps", type=int, default=2, help="alternating repetitions of each path")
    ap.add_argument("--gpus", default="1,2,4,8", help="runner counts of the table path (those visible)")
    ap.add_argument("--file-shape", default="256x200000x10", help="H x N x C of the host-resident file (fp16)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eps_search_table: needs a CUDA device")
    from coda_b200 import Dataset, TensorDataset
    from coda_b200.eps_search import hard_labels, modelpicker_eps_search
    from coda_b200.synth import synth
    print("card:", card(), "| visible GPUs:", torch.cuda.device_count(), flush=True)
    R, P, B = args.realisations, args.pool_size, args.budget
    for shape in args.shapes.split(","):
        H, C = (int(v) for v in shape.split("x"))
        preds, _ = synth(H, args.items, C, seed=0, device="cuda")
        table = hard_labels(TensorDataset(preds))
        del preds
        pools = np.stack([np.random.default_rng(r).permutation(args.items)[:P] for r in range(R)])
        search = lambda **kw: modelpicker_eps_search(table, epsilons=EPS, budget=B, seed=1, realisations=pools, **kw)
        warm = pools[:2, :64]
        modelpicker_eps_search(table, epsilons=EPS[:2], budget=8, seed=0, realisations=warm)   # module load, allocator
        times, same = {"global": [], "table": []}, True
        for _ in range(args.reps):
            t, g = timed(lambda: global_search(table, pools, 1, B))
            times["global"].append(t)
            t, res = timed(search)
            times["table"].append(t)
            same = same and all(np.array_equal(g[k], res[k]) for k in g)
        steps = len(EPS) * R * B
        line = {"H": H, "C": C, "N": args.items, "epsilons": len(EPS), "realisations": R, "pool": P, "budget": B,
                "global_s": [round(t, 3) for t in times["global"]], "table_s": [round(t, 3) for t in times["table"]],
                "table_steps_per_s": round(steps / min(times["table"]), 1), "bit_equal": same}
        print(json.dumps(line), flush=True)
        for k in (int(v) for v in args.gpus.split(",")):
            if k > torch.cuda.device_count():
                continue
            t, r = timed(lambda: search(gpus=k))
            assert all(np.array_equal(r[x], res[x]) for x in ("picks", "best", "pool_accuracies"))
            print(json.dumps({"H": H, "C": C, "gpus": k, "table_s": round(t, 3)}), flush=True)
        del table
    H, N, C = (int(v) for v in args.file_shape.split("x"))
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "task.pt")
        preds, _ = synth(H, N, C, seed=2, device="cuda")
        torch.save(preds.half().cpu(), path)
        del preds
        for k in (int(v) for v in args.gpus.split(",")):
            if k > torch.cuda.device_count():
                continue
            t, table = timed(lambda: hard_labels(Dataset(path, "cuda", host=True, shards=k if k > 1 else None)))
            print(json.dumps({"hard_labels_from_host_file": f"{H}x{N}x{C} fp16", "file_bytes": os.path.getsize(path),
                              "pieces": k, "seconds": round(t, 3)}), flush=True)
            del table


if __name__ == "__main__":
    main()
