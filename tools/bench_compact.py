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

``--large-c`` measures instead the compact path above C = 1000 (H = 64, N = 100000, C = 1000 / 2048 / 4096, K = 4 / 8):

* ``large_c_build``: CODA's construction on the compact slab, wall time and peak device memory, and the share of that
  peak the transposed-D scratch (H C^2 fp32) takes.
* ``large_c_stage``: each construction stage timed alone with CUDA events (scan, confusion, inverted index, marginals =
  D transpose + row sums + the full pass + pi_reduce); the scan both ways where both kernels run (``thread``: one
  thread per item, C <= 1599; ``warp``: one warp per item), which sets the switch point between them.
* ``large_c_refresh``: the per-step rank-1 refresh kernels under ``torch.profiler``: ``k_r1i_rows`` against its byte
  model (4 N C bytes of U read, one 32-byte sector per row for the column write, 16 N for R and the delta) and the slab
  scan ``k_pi_rank1_compact``.
* ``large_c_run``: ``run_steps`` steps/s with the inverted index (the default).
* ``large_c_scan``: the two scan kernels alone at C = 100 ... 1599 (K = 4, 8), to place the switch between them.
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


def _ms(torch, fn, repeats):
    """Mean milliseconds of fn() over ``repeats`` back-to-back calls, CUDA events, after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(repeats):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / repeats


def _kernel_us(torch, fn, calls, names):
    """Device time per call (us) of each kernel in ``names``, from torch.profiler over ``calls`` calls of fn()."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {n: 0.0 for n in names}
    for ev in prof.key_averages():
        for n in names:
            if n + "<" in ev.key or ev.key.startswith(n + "(") or ev.key == n:
                out[n] += getattr(ev, "device_time_total", getattr(ev, "cuda_time_total", 0.0))
    return {n: v / calls for n, v in out.items()}


def bench_scan_switch(torch, H, N, C, K, repeats):
    """The two scan kernels alone on one synthetic slab (``large_c_scan``): where the warp-per-item kernel overtakes."""
    import ctypes as ct
    from coda_b200 import _native as nat
    from coda_b200.synth import synth_compact
    ids, probs, _ = synth_compact(H, N, C, K, seed=C + K, device="cuda:0")
    lib = nat.load()
    P = ct.c_void_p
    hard = torch.empty((N, H), dtype=torch.int16, device="cuda:0")
    pseudo = torch.empty(N, dtype=torch.int32, device="cuda:0")
    dis = torch.empty(N, dtype=torch.uint8, device="cuda:0")
    ens = torch.empty((N, C), device="cuda:0")
    fl = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    s = torch.cuda.current_stream().cuda_stream
    row = dict(kind="large_c_scan", H=H, N=N, C=C, K=K)
    for name, kern in (("thread", 1), ("warp", 2)):
        row[f"{name}_ms"] = round(_ms(torch, lambda: nat_check(lib.coda_b200_scan_compact_kernel(
            P(ids.data_ptr()), P(probs.data_ptr()), N * K, H, N, C, K, P(hard.data_ptr()), P(pseudo.data_ptr()),
            P(dis.data_ptr()), P(ens.data_ptr()), P(fl.data_ptr()), kern, P(s))), repeats), 3)
    emit(**row)


def bench_large_c(torch, H, N, C, K, steps, warmup, repeats):
    import ctypes as ct
    from coda_b200 import CODA, CompactDataset, CompactSlab
    from coda_b200.synth import synth_compact
    dev = "cuda:0"
    ids, probs, labels = synth_compact(H, N, C, K, seed=C + K, device=dev)
    slab = CompactSlab(ids, probs, C)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    random.seed(0)
    sel = CODA(CompactDataset(slab, labels))
    torch.cuda.synchronize()
    ctor_s = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base
    dt_bytes = H * C * C * 4
    emit(kind="large_c_build", H=H, N=N, C=C, K=K, construct_s=round(ctor_s, 3), peak_GB=round(peak / 1e9, 3),
         DT_GB=round(dt_bytes / 1e9, 3), DT_share_of_peak=round(dt_bytes / peak, 3),
         slab_GB=round(6 * H * N * K / 1e9, 3))
    e = sel.engine
    # the device loop first: the stage timings below rewrite U and the column sums
    sel.run_steps(warmup, labels)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sel.run_steps(steps, labels)
    torch.cuda.synchronize()
    emit(kind="large_c_run", H=H, N=N, C=C, K=K, steps=steps, steps_per_s=round(steps / (time.perf_counter() - t0), 2),
         index=e.cidx is not None)
    P = ct.c_void_p
    s = torch.cuda.current_stream().cuda_stream
    lib = e.lib
    row = dict(kind="large_c_refresh", H=H, N=N, C=C, K=K)
    with e._on():
        if e.cidx is not None:
            ix = e.cidx
            us = _kernel_us(torch, lambda: lib.coda_b200_pi_rank1_index(
                P(ix["off"].data_ptr()), P(ix["ent"].data_ptr()), P(ix["rest"].data_ptr()), P(e.jvec.data_ptr()), H, N, C,
                P(e.sel.data_ptr()), ct.c_double(e.lr), e.fx_shift, P(e.terms.data_ptr()), P(ix["delta"].data_ptr()),
                P(e.U.data_ptr()), P(e.pisum.data_ptr()), P(e.flags.data_ptr()), P(s)), 20, ["k_r1i_rows", "k_r1i_scatter"])
            nbytes = 4 * N * C + 32 * N + 16 * N
            row.update(r1i_rows_us=round(us["k_r1i_rows"], 1), r1i_scatter_us=round(us["k_r1i_scatter"], 1),
                       r1i_rows_model_MB=round(nbytes / 1e6, 1),
                       r1i_rows_GBps=round(nbytes / max(us["k_r1i_rows"], 1e-9) / 1e3, 1),
                       r1i_rows_share_of_3_35TBps=round(nbytes / (max(us["k_r1i_rows"], 1e-9) * 1e-6) / HBM_PEAK, 3))
        cs = e.compact
        us = _kernel_us(torch, lambda: lib.coda_b200_pi_rank1_compact(
            P(cs.ids.data_ptr()), P(cs.probs.data_ptr()), e.model_stride, P(e.ens.data_ptr()), H, N, C, K,
            P(e.sel.data_ptr()), ct.c_double(e.lr), e.fx_shift, P(e.terms.data_ptr()), P(e.U.data_ptr()),
            P(e.pisum.data_ptr()), P(e.flags.data_ptr()), P(s)), 10, ["k_pi_rank1_compact"])
        row.update(pi_rank1_compact_us=round(us["k_pi_rank1_compact"], 1))
        emit(**row)
        st = dict(kind="large_c_stage", H=H, N=N, C=C, K=K)
        hard = torch.empty((N, H), dtype=torch.int16, device=dev)
        pseudo = torch.empty(N, dtype=torch.int32, device=dev)
        dis = torch.empty(N, dtype=torch.uint8, device=dev)
        ens = e.ens
        fl = torch.zeros(1, dtype=torch.int32, device=dev)
        outs = {}
        for name, kern in (("thread", 1), ("warp", 2)):
            if kern == 1 and C > 1599:
                continue
            st[f"scan_{name}_ms"] = round(_ms(torch, lambda: nat_check(lib.coda_b200_scan_compact_kernel(
                P(cs.ids.data_ptr()), P(cs.probs.data_ptr()), e.model_stride, H, N, C, K, P(hard.data_ptr()),
                P(pseudo.data_ptr()), P(dis.data_ptr()), P(ens.data_ptr()), P(fl.data_ptr()), kern, P(s))), repeats), 3)
            outs[name] = (hard.clone(), pseudo.clone(), dis.clone(), ens.clone())
        if len(outs) == 2:
            st["scan_kernels_bit_identical"] = all(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                                               b.view(torch.int32) if b.dtype == torch.float32 else b)
                                                   for a, b in zip(outs["thread"], outs["warp"]))
        del outs
        conf = torch.zeros(H * C * C + H * C, dtype=torch.int64, device=dev)
        st["confusion_ms"] = round(_ms(torch, lambda: nat_check(lib.coda_b200_confusion_compact(
            P(cs.ids.data_ptr()), P(cs.probs.data_ptr()), e.model_stride, P(pseudo.data_ptr()), H, N, C, K, e.fx_shift,
            P(conf.data_ptr()), P(conf[H * C * C:].data_ptr()), P(s))), repeats), 3)
        del conf
        torch.cuda.empty_cache()
        if e.cidx is not None:
            st["index_ms"] = round(_ms(torch, e._build_compact_index, 3), 3)
        st["marginals_ms"] = round(_ms(torch, e._marginals_full, 3), 3)
        emit(**st)
    sel.close()
    del sel, e, slab, ids, probs


def nat_check(rc):
    if rc != 0:
        from coda_b200 import _native as nat
        nat.check(rc, "bench_compact")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="small sizes (a rehearsal, not a measurement)")
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--large-c", action="store_true", help="the compact path at C = 1000, 2048, 4096 only")
    args = ap.parse_args()
    import torch
    from coda_b200 import _native as nat
    if not torch.cuda.is_available():
        raise SystemExit("bench_compact: needs a CUDA device")
    q = args.quick
    emit(kind="card", card=card(), torch_cuda_device=torch.cuda.get_device_name(0))
    if args.large_c:
        for C in (100, 200, 400, 800, 1000, 1599):
            for K in (4, 8):
                bench_scan_switch(torch, 64, 3000 if q else 100_000, C, K, 3 if q else args.repeats)
        for C in (1000, 2048, 4096):
            for K in (4, 8):
                try:
                    bench_large_c(torch, 64, 3000 if q else 100_000, C, K, 3 if q else 20, 2 if q else 5,
                                  3 if q else args.repeats)
                except Exception as ex:                    # a shape that fails is reported; the others still run
                    emit(kind="large_c_error", C=C, K=K, error=f"{type(ex).__name__}: {ex}"[:400])
                torch.cuda.empty_cache()
        emit(kind="card", card=card())
        return
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
