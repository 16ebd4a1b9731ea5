"""Steps/s of CODA with --prefilter-n, scoring only the sample against scoring every item, one JSON line on stdout.

    python tools/bench_prefilter.py [--H 256 --N 500000 --C 100] [--m 1000 10000 20000 30000 125000] [--steps 50]

One synthetic task (bench.py's cfg3 workload unless --H/--N/--C say otherwise) is generated once; for every m a CODA
selector is built with CODA_B200_PREFILTER_SCORING=sample and one with =full, and each is timed:
  * ``run_steps`` (the device loop, one CUDA-graph replay per step) and the public API loop (host oracle);
  * its scoring pass alone, CUDA events around ``--reps`` launches, twice: the sampled pass (sample.cu) over m random
    items, or the full pass (row_gains + gain_eig) over all N;
  * the bytes of its row cache (with the sampled pass: the template rows and the scratch) and the peak device memory.
The sampled pass's times are fitted as a + b * m (least squares); it beats the full pass below m* = (t_full - a) / b,
and R = N / m* is the engine's PREFILTER_ROW_COST_RATIO for this task.  The card's name and power limit are read in
the same run.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _time_scoring(sel, sample, reps):
    import torch
    e = sel.engine
    with e._on():
        if sample:
            e.sw["items"].copy_(torch.randperm(e.N, device=e.dev)[: e.pf_m].to(torch.int32))
            body = e._score_sample
        else:
            def body():
                e.scored = False
                e._score()
        body()
        out = []
        for _ in range(2):
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(reps):
                body()
            t1.record()
            t1.synchronize()
            out.append(t0.elapsed_time(t1) / reps)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--N", type=int, default=500_000)
    ap.add_argument("--C", type=int, default=100)
    ap.add_argument("--m", type=int, nargs="+", default=[1000, 10_000, 20_000, 30_000, 125_000])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--api-steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    sys.stdout.flush()
    real_stdout = os.dup(1)
    os.dup2(2, 1)

    import torch
    import coda_b200
    dev = torch.device("cuda", 0)
    ds = coda_b200.SyntheticDataset(args.H, args.N, args.C, seed=args.seed, device=dev)
    labels_host = ds.labels_host.numpy()
    labels_dev = ds.labels_host.to(dev)
    runs = []
    for m in args.m:
        for scoring in ("sample", "full"):
            os.environ["CODA_B200_PREFILTER_SCORING"] = scoring
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            random.seed(0)
            t = time.time()
            sel = coda_b200.CODA(ds, prefilter_n=m)
            torch.cuda.synchronize()
            t_init = time.time() - t
            e = sel.engine
            assert e.sample_scoring == (scoring == "sample")
            sel.run_steps(args.warmup, labels_dev)
            torch.cuda.synchronize()
            t = time.perf_counter()
            sel.run_steps(args.steps, labels_dev)
            torch.cuda.synchronize()
            loop_ms = (time.perf_counter() - t) * 1e3 / args.steps
            t = time.perf_counter()
            for _ in range(args.api_steps):
                idx, q = sel.get_next_item_to_label()
                sel.add_label(idx, int(labels_host[idx]), q)
                sel.get_best_model_prediction()
            torch.cuda.synchronize()
            api_ms = (time.perf_counter() - t) * 1e3 / args.api_steps
            score_ms = _time_scoring(sel, scoring == "sample", args.reps)
            cache = e.ph_cache.numel() * 4 + (e.sw["rows"].numel() * 4 if e.sw else 0)
            runs.append(dict(m=m, scoring=scoring, run_steps_per_s=1e3 / loop_ms, api_steps_per_s=1e3 / api_ms,
                             scoring_pass_ms=score_ms, heavy_rows_sampled=int(e.sw["nheavy"]) if e.sw else None,
                             row_cache_gb=cache / 2 ** 30, peak_gb=torch.cuda.max_memory_allocated(dev) / 2 ** 30,
                             init_s=t_init))
            n_heavy = e.n_heavy
            sel.close()
            del sel, e
    ms = np.array([r["m"] for r in runs if r["scoring"] == "sample"], dtype=np.float64)
    ts = np.array([np.mean(r["scoring_pass_ms"]) for r in runs if r["scoring"] == "sample"])
    b_fit, a_fit = np.polyfit(ms, ts, 1)
    t_full = float(np.mean([np.mean(r["scoring_pass_ms"]) for r in runs if r["scoring"] == "full"]))
    m_star = (t_full - a_fit) / b_fit
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        power = None
    line = {"metric": "prefilter_n steps/sec, sampled vs full scoring", "workload": dict(H=args.H, N=args.N, C=args.C),
            "runs": runs, "fit_ms": dict(a=float(a_fit), b_per_item=float(b_fit), full=t_full),
            "crossover_m": float(m_star), "row_cost_ratio_R": float(args.N / m_star), "n_heavy": n_heavy,
            "device": torch.cuda.get_device_name(dev), "power_limit": power, "steps": args.steps,
            "api_steps": args.api_steps}
    sys.stdout.flush()
    os.write(real_stdout, (json.dumps(line) + "\n").encode())


if __name__ == "__main__":
    main()
