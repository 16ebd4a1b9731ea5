"""ModelPicker steps per second of the epsilon grid search: the batched device search (coda_b200.eps_search) against
one ``ModelPicker(...).run_steps`` per run, construction included, on synthetic tasks.

    python tools/bench_eps_search.py [--realisations 1000] [--pool-size 1000] [--budget 1000] [--per-run 4]

The default grid is the reference script's (15 epsilons x 1000 realisations x pool 1000 x budget 1000) at
H = 64 / C = 10 and H = 256 / C = 100.  The per-run path times ``--per-run`` runs and extrapolates to the grid.  Prints
the card and its power limit with the numbers, and the byte model of the kernel: the pool's hard rows (P x H x 2 bytes)
one step reads, once per CTA for all the epsilons it carries, against once per run on the per-run path.
"""
import argparse
import json
import os
import subprocess
import sys
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--realisations", type=int, default=1000)
    ap.add_argument("--pool-size", type=int, default=1000)
    ap.add_argument("--budget", type=int, default=1000)
    ap.add_argument("--items", type=int, default=20000, help="N of the synthetic task")
    ap.add_argument("--per-run", type=int, default=4, help="runs timed on the per-run path")
    ap.add_argument("--shapes", default="64x10,256x100", help="H x C of the synthetic tasks")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eps_search: needs a CUDA device")
    from coda_b200 import ModelPicker, TensorDataset, _native as nat
    from coda_b200.eps_search import eps_search_run_key, modelpicker_eps_search
    from coda_b200.synth import synth
    print("card:", card(), flush=True)
    E, R, P, B = len(EPS), args.realisations, args.pool_size, args.budget
    for shape in args.shapes.split(","):
        H, C = (int(v) for v in shape.split("x"))
        preds, _ = synth(H, args.items, C, seed=0, device="cuda")
        ds = TensorDataset(preds)
        plan = np.zeros(5, dtype=np.int64)
        nat.check(nat.load().coda_b200_mp_runs_plan(H, E, P, R, B, plan.ctypes.data), "mp_runs_plan")
        # warm-up: module load, allocator
        np.random.seed(0)
        modelpicker_eps_search(ds, epsilons=EPS[:2], iterations=2, pool_size=min(P, 64), budget=8, seed=0)
        np.random.seed(1)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = modelpicker_eps_search(ds, epsilons=EPS, iterations=R, pool_size=P, budget=B, seed=1)
        torch.cuda.synchronize()
        t_batch = time.perf_counter() - t0
        steps = E * R * B
        # per-run path on the first runs of the same search, construction included
        lab = torch.as_tensor(res["labels"], device="cuda")
        n = max(1, args.per_run)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(n):
            e, r = i % E, i // E
            pool = torch.as_tensor(res["realisations"][r], device="cuda")
            sel = ModelPicker(TensorDataset(preds[:, pool].contiguous()), epsilon=EPS[e])
            sel.run_steps(B, lab[pool], seed=eps_search_run_key(res["seed"], e, r))
            sel.history()
            sel.close()
        torch.cuda.synchronize()
        t_run = (time.perf_counter() - t0) / n
        row_bytes = P * H * 2
        line = {"H": H, "C": C, "N": args.items, "epsilons": E, "realisations": R, "pool": P, "budget": B,
                "runs_per_cta": int(plan[0]), "eps_blocks": int(plan[1]), "realisations_per_launch": int(plan[2]),
                "batched_s": round(t_batch, 3), "batched_steps_per_s": round(steps / t_batch, 1),
                "per_run_s": round(t_run, 4), "per_run_steps_per_s": round(B / t_run, 1),
                "per_run_grid_s_extrapolated": round(t_run * E * R, 1),
                # hard-row bytes one step reads per realisation with every pool item unlabeled (an upper bound)
                "row_bytes_per_step_batched": row_bytes * int(plan[1]), "row_bytes_per_step_per_run": row_bytes * E}
        print(json.dumps(line), flush=True)
        del ds, preds, res


if __name__ == "__main__":
    main()
