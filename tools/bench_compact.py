"""Compact top-K slabs built on the device: the compaction kernel, a file -> pieces load, CODA on the compacted task
against the dense one, and how far the compacted run drifts.  One JSON line per measurement on stdout.

    python tools/bench_compact.py [--quick]

* ``kernel``: ``coda_b200_compact_build`` alone on a device slab, timed with CUDA events over ``--repeats`` launches;
  dense GB/s = the dense bytes read once (H*N*C*s, s = 4 or 2) plus the 6*K*H*N bytes written, over kernel time, and
  its share of the H100 SXM data-sheet 3.35 TB/s.  fp32 and fp16 at C = 100 and 1000, K = 4 and 8.
* ``load``: ``load_compact`` of a freshly written dense file (file bytes over wall time).  The file was just written, so
  its pages are likely in the host page cache: this is not a cold-disk read.
* ``run``: ``CODA.run_steps`` steps/s and peak device memory on the compacted task and on the dense task, one GPU.
* ``drift``: the compacted run against the dense run from the same seed: how many of the first 100 picks agree, the
  largest P(best) difference after them, and each run's final regret against the dense true losses.  The data are
  synthetic (``coda_b200.synth``); their tail classes are not real softmax tails, so this says little about real tasks.
The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_PEAK = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                                    # the measurement stands; say why the card is unknown
        return f"unknown ({e})"


def emit(**kw):
    print(json.dumps(kw), flush=True)


def bench_kernel(torch, nat, H, N, C, K, dtype, repeats):
    import ctypes as ct
    x = torch.rand(H, N, C, device="cuda:0").softmax(-1).to(dtype)
    ids = torch.empty(H, N, K, dtype=torch.int16, device="cuda:0")
    probs = torch.empty(H, N, K, dtype=torch.float32, device="cuda:0")
    dropped = torch.zeros(H, device="cuda:0")
    flat = torch.zeros(H, dtype=torch.int64, device="cuda:0")
    flags = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    lib = nat.load()
    args = (ct.c_void_p(x.data_ptr()), nat.slab_format(dtype), N * C, H, N, C, K, ct.c_void_p(ids.data_ptr()),
            ct.c_void_p(probs.data_ptr()), N * K, ct.c_void_p(dropped.data_ptr()), ct.c_void_p(flat.data_ptr()),
            ct.c_void_p(flags.data_ptr()), ct.c_void_p(torch.cuda.current_stream().cuda_stream))
    for _ in range(3):
        nat.check(lib.coda_b200_compact_build(*args), "compact_build")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(repeats):
        lib.coda_b200_compact_build(*args)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / repeats
    nbytes = H * N * C * x.element_size() + 6 * K * H * N
    emit(kind="kernel", H=H, N=N, C=C, K=K, dtype=str(dtype).replace("torch.", ""), ms=round(ms, 4),
         GBps=round(nbytes / ms / 1e6, 1), share_of_3_35TBps=round(nbytes / (ms / 1e3) / HBM_PEAK, 3))
    del x, ids, probs


def bench_load(torch, H, N, C, K, tmpdir):
    from coda_b200.datasets import load_compact
    path = os.path.join(tmpdir, "task.pt")
    torch.save(torch.rand(H, N, C, generator=torch.Generator().manual_seed(0)).softmax(-1), path)
    nbytes = os.path.getsize(path)
    load_compact(path, "cuda:0", K, chunk_bytes=1 << 20)        # warm the kernels and the pinned allocator
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    slab = load_compact(path, "cuda:0", K)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    emit(kind="load", H=H, N=N, C=C, K=K, file_GB=round(nbytes / 1e9, 3), load_s=round(s, 3),
         file_GBps=round(nbytes / s / 1e9, 2), page_cache="likely warm (file just written)", pieces=1)
    del slab
    os.remove(path)


def _run(torch, CODA, TensorDataset, preds, labels, steps, warmup):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    random.seed(0)
    sel = CODA(TensorDataset(preds, labels))
    sel.run_steps(warmup, labels)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sel.run_steps(steps, labels)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base
    return steps / dt, peak


def bench_run(torch, H, N, C, K, steps, warmup):
    from coda_b200 import CODA, CompactSlab, TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, 0)
    dense = preds.to("cuda:0")
    lab = labels.to("cuda:0")
    comp = CompactSlab.from_dense(dense, K)
    sps_c, peak_c = _run(torch, CODA, TensorDataset, comp, lab, steps, warmup)
    sps_d, peak_d = _run(torch, CODA, TensorDataset, dense, lab, steps, warmup)
    emit(kind="run", H=H, N=N, C=C, K=K, steps=steps, compact_steps_per_s=round(sps_c, 2),
         dense_steps_per_s=round(sps_d, 2), compact_peak_GB=round(peak_c / 1e9, 3), dense_peak_GB=round(peak_d / 1e9, 3),
         compact_slab_GB=round(H * N * K * 6 / 1e9, 3), dense_slab_GB=round(H * N * C * 4 / 1e9, 3))


def bench_drift(torch, H, N, C, K, steps):
    from coda.options import LOSS_FNS
    from coda_b200 import CODA, CompactSlab, Oracle, TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, 1)
    dense = preds.to("cuda:0")
    lab = labels.to("cuda:0")
    comp = CompactSlab.from_dense(dense, K)
    tl = Oracle(TensorDataset(dense, lab), loss_fn=LOSS_FNS["acc"]).true_losses(dense)
    out = {}
    for name, slab in (("dense", dense), ("compact", comp)):
        random.seed(0)
        sel = CODA(TensorDataset(slab, lab))
        sel.run_steps(steps, lab, record_best=True)
        out[name] = (sel.history()[0].tolist(), sel.get_pbest().float().cpu(), int(sel.best_history()[0][-1]))
    agree = sum(a == b for a, b in zip(out["dense"][0], out["compact"][0]))
    same_prefix = next((i for i, (a, b) in enumerate(zip(out["dense"][0], out["compact"][0])) if a != b), steps)
    emit(kind="drift", H=H, N=N, C=C, K=K, steps=steps, picks_agree=agree, identical_prefix=same_prefix,
         max_pbest_diff=float((out["dense"][1] - out["compact"][1]).abs().max()),
         dense_final_regret=float(tl[out["dense"][2]] - tl.min()),
         compact_final_regret=float(tl[out["compact"][2]] - tl.min()),
         flat_rows=int(comp.compaction["flat_rows"].sum()), dropped_max=float(comp.compaction["dropped_max"].max()),
         note="synthetic scores: their tails are not real softmax tails")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes (a rehearsal, not a measurement)")
    ap.add_argument("--repeats", type=int, default=20)
    args = ap.parse_args()
    import torch
    from coda_b200 import _native as nat
    if not torch.cuda.is_available():
        raise SystemExit("bench_compact: needs a CUDA device")
    q = args.quick
    emit(kind="card", card=card(), torch_cuda_device=torch.cuda.get_device_name(0))
    for C in (100, 1000):
        N = (2000 if q else 200_000) * 100 // C
        for dtype in (torch.float32, torch.float16):
            for K in (4, 8):
                bench_kernel(torch, nat, 64, N, C, K, dtype, 3 if q else args.repeats)
    with tempfile.TemporaryDirectory() as tmp:
        bench_load(torch, 32, 2000 if q else 100_000, 100, 4, tmp)
    bench_run(torch, 64, 2000 if q else 100_000, 100, 4, 10 if q else 100, 3 if q else 10)
    bench_drift(torch, 64, 2000 if q else 20_000, 100, 4, 100)
    emit(kind="card", card=card())


if __name__ == "__main__":
    main()
