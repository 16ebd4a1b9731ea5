"""Steps/s of one competing selector (coda_b200.baselines) or of CODA, one JSON line on stdout.

    python tools/bench_baselines.py --method {iid,uncertainty,activetesting,vma,model_picker,coda} [--steps 100] [--warmup 10]
        [--shards S] [--gpus G] [--compact K] [--loop {api,device}] [--q {eig,iid,uncertainty}] [--prefilter-n K]
        [--tie-rule {first,philox,reference}]
    python -m torch.distributed.run --nproc-per-node 8 tools/bench_baselines.py --method model_picker --N 1000000

--loop device times ``run_steps`` (one CUDA-graph replay per step and shard, the oracle's labels on the device) instead
of the public API loop, and reports the final and cumulative regret of the timed steps from ``best_history()`` and the
true accuracy losses of the models (Oracle.true_losses).  Not under torchrun.  --method coda runs CODA with its default
arguments unless --q / --prefilter-n name its other acquisitions (coda.py:215-224, 287-295); its device loop is
``run_steps(..., record_best=True)``, the graph that also records each step's best model.  --tie-rule picks run_steps'
tie rule: ``first`` / ``reference`` for CODA, ``philox`` / ``reference`` (torch's own generators, mirrored on the
device) for the five competing selectors; the default is each one's default.

--shards / --gpus split the task over in-process N-range shards (shards may share a GPU); under torchrun every rank
holds its own N-range and rank 0 prints the line.  --compact K generates the task directly as a top-K compact slab
(SyntheticCompactDataset).

One step = get_next_item_to_label() -> oracle(idx) -> add_label() -> get_best_model_prediction() through the public API
with a host oracle (reference main.py:91-94), on the synthetic cfg3 workload of bench.py (256 x 5e5 x 100, a 51 GB
slab) unless --H/--N/--C say otherwise.  Also reported: construction time (including the slab scan), the card and its
power limit read in the same run, and for ModelPicker the algorithmic bytes of its per-step entropy pass.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

METHODS = {"iid": "IID", "uncertainty": "Uncertainty", "activetesting": "ActiveTesting", "vma": "VMA",
           "model_picker": "ModelPicker", "coda": "CODA"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--method", required=True, choices=sorted(METHODS))
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--N", type=int, default=500_000)
    ap.add_argument("--C", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--dense", action="store_true", help="worst-case synthetic slab (wrong class uniform)")
    ap.add_argument("--shards", type=int, default=None, help="in-process N-range shards (default: one)")
    ap.add_argument("--gpus", type=int, default=None, help="GPUs the in-process shards are spread over")
    ap.add_argument("--compact", type=int, default=0, metavar="K", help="top-K compact slab instead of a dense one")
    ap.add_argument("--loop", choices=["api", "device"], default="api", help="public API loop or run_steps")
    ap.add_argument("--q", choices=["eig", "iid", "uncertainty"], default="eig", help="CODA's acquisition (--method coda)")
    ap.add_argument("--prefilter-n", type=int, default=0, help="CODA's random subsample of the candidates (--method coda)")
    ap.add_argument("--tie-rule", choices=["first", "philox", "reference"], default=None,
                    help="run_steps' tie rule (--loop device): first | reference for coda, philox | reference otherwise")
    args = ap.parse_args()
    if args.method != "coda" and (args.q != "eig" or args.prefilter_n):
        raise SystemExit("bench_baselines: --q and --prefilter-n are options of --method coda")
    if args.tie_rule is not None and args.loop != "device":
        raise SystemExit("bench_baselines: --tie-rule is an option of --loop device")
    rules = ("first", "reference") if args.method == "coda" else ("philox", "reference")
    args.tie_rule = args.tie_rule or rules[0]
    if args.tie_rule not in rules:
        raise SystemExit(f"bench_baselines: --method {args.method} takes --tie-rule {' or '.join(rules)}")
    if args.steps + args.warmup >= args.N:
        raise SystemExit("bench_baselines: steps + warmup must stay below the number of items")
    # stdout carries exactly one JSON line
    sys.stdout.flush()
    real_stdout = os.dup(1)
    os.dup2(2, 1)

    import torch
    import coda_b200
    from coda.options import LOSS_FNS
    H, N, C = args.H, args.N, args.C
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", 0)))
    torch.cuda.set_device(dev)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    if args.compact:
        ds = coda_b200.SyntheticCompactDataset(H, N, C, K=args.compact, seed=args.seed, device=dev, rank=rank, world=world)
    else:
        ds = coda_b200.SyntheticDataset(H, N, C, seed=args.seed, device=dev, dense=args.dense, rank=rank, world=world)
    labels = ds.labels_host.numpy()
    torch.cuda.synchronize()
    random.seed(0)
    torch.manual_seed(0)
    cls = getattr(coda_b200, METHODS[args.method])
    kw = dict(shards=args.shards, gpus=args.gpus)
    if args.q != "eig" or args.prefilter_n:
        kw.update(q=args.q, prefilter_n=args.prefilter_n)
    t = time.time()
    sel = cls(ds, **kw) if args.method in ("model_picker", "coda") else cls(ds, LOSS_FNS["acc"], **kw)
    torch.cuda.synchronize()
    t_init = time.time() - t

    def step():
        idx, q = sel.get_next_item_to_label()
        sel.add_label(idx, int(labels[idx]), q)
        return int(sel.get_best_model_prediction())

    regret = None
    if args.loop == "device":
        labels_dev = ds.labels_host.to(dev)
        if args.method == "coda":
            loop_kw = dict(record_best=True, tie_rule=args.tie_rule)
        elif args.tie_rule == "reference":
            loop_kw = dict(tie_rule="reference")           # draws from torch's generators, seeded above
        else:
            loop_kw = dict(seed=args.seed)
        sel.run_steps(args.warmup, labels_dev, **loop_kw)
        torch.cuda.synchronize()
        t = time.perf_counter()
        sel.run_steps(args.steps, labels_dev, **loop_kw)
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t) * 1e3 / args.steps
        best, _ties = sel.best_history()
        # [N][H] arg-max class of every model (the slab scan)
        hard = sel._cat("hard") if args.method == "coda" else sel.hard
        true_losses = torch.zeros(H, dtype=torch.float64, device=dev)
        for lo in range(0, hard.shape[0], 65536):         # accuracy loss of every model over all items
            h = hard[lo:lo + 65536].to(torch.int64) & 0xFFFF
            true_losses += (h != labels_dev[lo:lo + 65536, None]).sum(0).double()
        true_losses = (true_losses / hard.shape[0]).cpu().numpy()
        r = true_losses[best[args.warmup:]] - true_losses.min()
        regret = {"final": float(r[-1]), "cumulative": float(r.sum())}
    else:
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t) * 1e3 / args.steps
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        power = None
    shards = getattr(sel, "states", None) or sel.engines
    line = {"metric": "baseline acquisition steps/sec", "method": args.method, "value": 1e3 / ms, "unit": "steps/s",
            "ms_per_step": ms, "steps": args.steps, "warmup": args.warmup, "init_s": t_init,
            "workload": dict(H=H, N=N, C=C, dense=bool(args.dense), compact_k=args.compact, seed=args.seed),
            "shards": len(shards) * world, "processes": world, "gpus": len({st.dev for st in shards}) * world,
            "device": torch.cuda.get_device_name(dev), "power_limit": power,
            "loop": "public API, host oracle (main.py:91-94)"}
    if "q" in kw:
        line["coda"] = dict(q=args.q, prefilter_n=args.prefilter_n)
    if args.loop == "device":
        line["loop"] = "device: run_steps, one CUDA-graph replay per step and shard"
        line["regret"] = regret
        line["tie_rule"] = args.tie_rule
        line["tie_steps"] = int(sel.history()[2][args.warmup:].sum())
        if args.method != "coda":
            line["best_tie_steps"] = int(sel.best_history()[1][args.warmup:].sum())
    if args.method == "model_picker":
        nbytes = 2 * H * N + 2 * N + 4 * N          # hard rows + labeled / disagree masks + entropies, per step
        line["bytes_per_step"] = nbytes
        line["hbm_fraction_of_3.35TBps"] = nbytes / (ms * 1e-3) / 3.35e12
    sel.close()
    sys.stdout.flush()
    if rank == 0:
        os.write(real_stdout, (json.dumps(line) + "\n").encode())
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
