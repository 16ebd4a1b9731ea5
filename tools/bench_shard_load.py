"""Load a prediction slab as N-range pieces (``coda_b200.datasets.load_sharded``) and run the true-loss pass on them;
one JSON line on stdout.

    python tools/bench_shard_load.py --H 256 --N 200000 --C 100 --dtype f32 --shards 2 [--path task.pt] [--repeats 20]

Writes a synthetic (H, N, C) ``.pt`` task of the given dtype to a temporary directory (or reads ``--path``), then
reports the load time and GB/s per device and overall (file bytes over wall time; the first read of a freshly written
file may come from the page cache), and the true-loss pass (``Oracle.true_losses`` on the pieces, accuracy loss) timed
with CUDA events: its algorithmic bytes, s*H*N_i*C + 8*N_i per piece launch (s = 4 or 2), and GB/s against the H100
SXM data-sheet 3.35 TB/s.  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DTYPES = {"f32": "float32", "f16": "float16", "bf16": "bfloat16"}
HBM_PEAK = 3.35e12


def pass_bytes(slab):
    """The true-loss pass's algorithmic bytes: every piece's scores once at their stored width, its labels once."""
    H, _, C = slab.shape
    s = slab.element_size()
    return sum(s * H * p.shape[1] * C + 8 * p.shape[1] for p in slab.pieces)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--N", type=int, default=100_000)
    ap.add_argument("--C", type=int, default=100)
    ap.add_argument("--dtype", default="f32", choices=sorted(DTYPES))
    ap.add_argument("--keep-dtype", action="store_true")
    ap.add_argument("--shards", type=int, default=1)
    ap.add_argument("--gpus", type=int, default=None)
    ap.add_argument("--chunk-mb", type=int, default=64)
    ap.add_argument("--path", default=None)
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()

    import torch
    from coda.options import LOSS_FNS
    from coda_b200 import Oracle, TensorDataset
    from coda_b200.datasets import load_sharded
    if not torch.cuda.is_available():
        raise SystemExit("bench_shard_load: needs a CUDA device")
    tmp = None
    path = args.path
    if path is None:
        tmp = tempfile.TemporaryDirectory()
        path = os.path.join(tmp.name, "task.pt")
        g = torch.Generator().manual_seed(0)
        torch.save(torch.rand(args.H, args.N, args.C, generator=g).to(getattr(torch, DTYPES[args.dtype])), path)
    file_bytes = os.path.getsize(path)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    slab = load_sharded(path, "cuda:0", args.keep_dtype, shards=args.shards, gpus=args.gpus,
                        chunk_bytes=args.chunk_mb << 20)
    for d in {p.device for p in slab.pieces}:
        torch.cuda.synchronize(d)
    load_s = time.perf_counter() - t0
    H, N, C = slab.shape
    per_dev = {}
    for p in slab.pieces:
        per_dev[str(p.device)] = per_dev.get(str(p.device), 0) + p.shape[1] * H * C
    src_esz = file_bytes / max(1, H * N * C)
    labels = torch.randint(0, C, (N,), device="cuda:0")
    ora = Oracle(TensorDataset(slab, labels), loss_fn=LOSS_FNS["acc"])
    for _ in range(3):
        ora.true_losses(slab)
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t1 = time.perf_counter()
    ev0.record()
    for _ in range(args.repeats):
        ora.true_losses(slab)
    ev1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t1) / args.repeats
    pass_s = ev0.elapsed_time(ev1) / 1e3 / args.repeats
    nbytes = pass_bytes(slab)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                    # the measurement stands; say why the card is unknown
        card = f"unknown ({e})"
    line = {
        "H": H, "N": N, "C": C, "file_dtype": args.dtype, "slab_dtype": str(slab.dtype).replace("torch.", ""),
        "shards": len(slab.pieces), "devices": len(per_dev), "chunk_mb": args.chunk_mb,
        "load_s": round(load_s, 4), "load_GBps": round(file_bytes / load_s / 1e9, 3),
        "load_GBps_per_device": {d: round(n * src_esz / load_s / 1e9, 3) for d, n in per_dev.items()},
        "true_loss_ms": round(pass_s * 1e3, 4), "true_loss_wall_ms": round(wall * 1e3, 4),
        "true_loss_bytes": nbytes, "true_loss_GBps": round(nbytes / pass_s / 1e9, 1),
        "true_loss_share_of_3.35TBps": round(nbytes / pass_s / HBM_PEAK, 3),
        "card": card, "torch_cuda_device": torch.cuda.get_device_name(0),
    }
    print(json.dumps(line), flush=True)
    if tmp is not None:
        tmp.cleanup()


if __name__ == "__main__":
    main()
