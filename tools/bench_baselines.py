"""Steps/s of one competing selector (coda_b200.baselines), one JSON line on stdout.

    python tools/bench_baselines.py --method {iid,uncertainty,activetesting,vma,model_picker} [--steps 100] [--warmup 10]
        [--shards S] [--gpus G] [--compact K]
    python -m torch.distributed.run --nproc-per-node 8 tools/bench_baselines.py --method model_picker --N 1000000

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
           "model_picker": "ModelPicker"}


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
    args = ap.parse_args()
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
    t = time.time()
    sel = cls(ds, **kw) if args.method == "model_picker" else cls(ds, LOSS_FNS["acc"], **kw)
    torch.cuda.synchronize()
    t_init = time.time() - t

    def step():
        idx, q = sel.get_next_item_to_label()
        sel.add_label(idx, int(labels[idx]), q)
        return int(sel.get_best_model_prediction())

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
    line = {"metric": "baseline acquisition steps/sec", "method": args.method, "value": 1e3 / ms, "unit": "steps/s",
            "ms_per_step": ms, "steps": args.steps, "warmup": args.warmup, "init_s": t_init,
            "workload": dict(H=H, N=N, C=C, dense=bool(args.dense), compact_k=args.compact, seed=args.seed),
            "shards": len(sel.states) * world, "processes": world, "gpus": len({st.dev for st in sel.states}) * world,
            "device": torch.cuda.get_device_name(dev), "power_limit": power,
            "loop": "public API, host oracle (main.py:91-94)"}
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
