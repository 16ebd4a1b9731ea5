"""Measure CODA on one GPU from a dense slab kept in host memory (``HostSlab``), one JSON line per run:

    python tools/bench_host_slab.py [--H 256] [--N 0] [--C 100] [--steps 50] [--compare] [--pieces 1]

``--N 0`` takes the largest N <= 1e6 whose slab and host shadow slots fit in MemAvailable (/proc/meminfo), or refuses
with the numbers.  A line reports the card and its power limit, the construction time of each pass, ``run_steps`` and
API (end-to-end) steps/s, the device slots S, the host-slot bytes, the host columns staged per step and the time and
rate of ``k_host_stage``.  ``--compare`` also runs the same slab device-resident, alternating the two placements, and
checks their histories and final states byte for byte (``CODA_B200_SHADOW_MODELS`` is set so that host columns are
staged).

``--pieces k`` (k > 1) holds the host slab as k N-range pieces (``ShardedHostSlab``, the ranges and devices of
``load_host(shards=k)``) over the visible GPUs, and the device-resident twin as the same k ``ShardedSlab`` pieces; the
host columns per step and the ``k_host_stage`` time per step are then summed over the pieces."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def mem_available():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    return 0


def pick_n(H, C, want):
    avail = mem_available()
    for n in ([want] if want else [1_000_000, 750_000, 500_000, 250_000, 100_000]):
        need = int(1.5 * H * n * C * 4)          # the slab plus, at worst, half of it in host slots
        if need < 0.9 * avail:
            return n, avail
    sys.exit(f"bench_host_slab: no N fits: {avail / 2**30:.1f} GiB available, "
             f"{1.5 * H * (want or 100_000) * C * 4 / 2**30:.1f} GiB needed")


def timed_engine_phases(times):
    from coda_b200 import engine as E
    for name in ("construct_scan", "construct_posterior", "construct_tables"):
        orig = getattr(E.Engine, name)

        def wrap(self, *a, _o=orig, _n=name, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = _o(self, *a, **kw)
            torch.cuda.synchronize()
            times[_n] = times.get(_n, 0.0) + time.perf_counter() - t0
            return r
        setattr(E.Engine, name, wrap)


def dataset(preds, labels, host, chunk, pieces):
    from coda_b200 import HostDataset, HostSlab, ShardedHostSlab, ShardedSlab, TensorDataset
    from coda_b200.datasets import piece_plan
    if pieces == 1:
        if host:
            return HostDataset(HostSlab(preds, "cuda:0", chunk_items=chunk), labels.cuda())
        return TensorDataset(preds.cuda(), labels.cuda())
    ngpus = torch.cuda.device_count()
    plan = piece_plan(int(preds.shape[1]), pieces, min(pieces, ngpus), 0, ngpus)
    if host:
        slab = ShardedHostSlab([HostSlab(preds[:, lo:hi], torch.device("cuda", d), chunk_items=chunk)
                                for lo, hi, d in plan])
    else:
        slab = ShardedSlab([preds[:, lo:hi].contiguous().to(torch.device("cuda", d)) for lo, hi, d in plan])
    return TensorDataset(slab, labels.cuda())


def host_cols(sel):
    return sum(int(e.host_cols.item()) for e in sel.engines if e.host_cols is not None)


def run(preds, labels, host, steps, chunk, pieces=1):
    from coda_b200 import CODA
    import random
    random.seed(0)
    times = {}
    t0 = time.perf_counter()
    ds = dataset(preds, labels, host, chunk, pieces)
    sel = CODA(ds)
    torch.cuda.synchronize()
    times["construct_total"] = time.perf_counter() - t0
    e = sel.engine
    lab = labels.cuda()
    out = {"placement": "host" if host else "device", "construct_s": {k: round(v, 3) for k, v in times.items()}}
    if pieces > 1:
        out.update(pieces=pieces, piece_devices=[x.dev.index for x in sel.engines])
    c0 = host_cols(sel)
    # API path (end to end, graphs on)
    for _ in range(3):
        i, q = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), q)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        i, q = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), q)
        sel.get_best_model_prediction()
    torch.cuda.synchronize()
    out["api_steps_per_s"] = round(steps / (time.perf_counter() - t0), 2)
    sel.run_steps(2, lab)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sel.run_steps(steps, lab)
    sel.history()
    out["run_steps_per_s"] = round(steps / (time.perf_counter() - t0), 2)
    idx, q, _t = sel.history()
    digest = (idx.tobytes(), q.tobytes(), sel.pi_hat_xi.cpu().numpy().tobytes(), sel.dirichlets.cpu().numpy().tobytes())
    if host:
        cols = host_cols(sel) - c0
        engines = sel.engines
        if pieces == 1:
            out.update(S=e.n_shadow, n_host=e.n_host)
        else:
            out.update(S=[x.n_shadow for x in engines], n_host=[x.n_host for x in engines])
        out.update(host_slot_bytes=sum(x.n_host * x.C * x.shadow_cs * x.esz for x in engines),
                   host_cols_per_step=round(cols / (2 * steps + 5), 2))
        # k_host_stage alone: eager steps with every launch of the entry point bracketed by events
        for x in engines:
            x.use_graph = False
            x.start_profile(only={"coda_b200_host_stage"})
        staged = -sum(int(x.host_cols.item()) * x.shadow_cs * x.esz for x in engines)
        for _ in range(10):
            i, q = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), q)
        profs = [x.stop_profile().get("coda_b200_host_stage", (0, 0.0, 0.0)) for x in engines]
        staged += sum(int(x.host_cols.item()) * x.shadow_cs * x.esz for x in engines)
        ms = sum(p[1] for p in profs)
        out["host_stage_ms_per_step"] = round(ms / max(1, profs[0][0]), 4)
        out["host_stage_GBps"] = round(staged / max(1e-9, ms * 1e-3) / 1e9, 2)
    sel.close()
    return out, digest


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--N", type=int, default=0)
    ap.add_argument("--C", type=int, default=100)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--chunk-items", type=int, default=None)
    ap.add_argument("--shadow-models", type=int, default=None)
    ap.add_argument("--compare", action="store_true")
    ap.add_argument("--pieces", type=int, default=1)
    a = ap.parse_args()
    if a.shadow_models is not None:
        os.environ["CODA_B200_SHADOW_MODELS"] = str(a.shadow_models)
    from coda_b200.synth import synth
    N, avail = pick_n(a.H, a.C, a.N)
    times = {}
    timed_engine_phases(times)
    preds, labels = synth(a.H, N, a.C, 0)
    base = {"card": card(), "H": a.H, "N": N, "C": a.C, "mem_available_gib": round(avail / 2**30, 1),
            "shadow_models_cap": os.environ.get("CODA_B200_SHADOW_MODELS")}
    order = [True, False, True, False] if a.compare else [True]
    digests = {}
    for host in order:
        times.clear()
        out, dig = run(preds.contiguous(), labels, host, a.steps, a.chunk_items, a.pieces)
        out["construct_s"].update({k: round(v, 3) for k, v in times.items()})
        digests.setdefault(host, dig)
        if a.compare:
            other = digests.get(not host)
            out["same_as_other_placement"] = None if other is None else dig == other
        print(json.dumps({**base, **out}), flush=True)


if __name__ == "__main__":
    main()
