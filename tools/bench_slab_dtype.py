"""CODA steps/s on one GPU with the prediction slab stored as fp32, fp16 or bf16; one JSON line on stdout.

    python tools/bench_slab_dtype.py --dtype {f32,f16,bf16} [--N 1000000] [--steps 300] [--warmup 10] [--dump-outputs DIR]
    python tools/bench_slab_dtype.py --dtype f16 --N 250000 --compare-widened

The synthetic cfg3 task of bench.py (256 x 5e5 x 100) unless --H/--N/--C say otherwise; --N 1000000 is cfg3 at its full
size (102.4 GB as fp32, 51.2 GB as fp16).  A 16-bit slab is generated block by block in its width (synth(dtype=)), so
the fp32 slab never exists.  A configuration whose slab, U and ensemble sums do not fit the device stops before it
allocates anything.

Reported: the host-free graph loop (`value`, CUDA events around run_steps), the public API loop with a host oracle
(`e2e`), construction time, the models in the class-major shadow, k_pi_rank1's time from an eager profile, and the card
and its power limit read in the same run.  --dump-outputs writes the graph loop's picks, the final EIG vector and P(best)
as .npy.  --compare-widened also runs the fp32 widening of the same 16-bit slab (both must fit at once) and reports
whether picks, EIG and P(best) are bit-identical.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

DTYPES = ("f32", "f16", "bf16")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="f32", choices=DTYPES)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--e2e-steps", type=int, default=100)
    ap.add_argument("--H", type=int, default=256)
    ap.add_argument("--N", type=int, default=500_000)
    ap.add_argument("--C", type=int, default=100)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    ap.add_argument("--compare-widened", action="store_true")
    args = ap.parse_args()
    if args.steps + args.warmup + args.e2e_steps + 64 >= args.N:
        raise SystemExit("bench_slab_dtype: steps must stay below the number of items")
    sys.stdout.flush()
    real_stdout = os.dup(1)                  # stdout carries exactly one JSON line
    os.dup2(2, 1)

    import numpy as np
    import torch
    from coda_b200 import CODA, SyntheticDataset, TensorDataset
    dt = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}[args.dtype]
    H, N, C = args.H, args.N, args.C
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    need = H * N * C * dt.itemsize + 8 * N * C
    if args.compare_widened:
        need += 4 * H * N * C
    have = torch.cuda.get_device_properties(dev).total_memory
    if need > have:
        raise SystemExit(f"bench_slab_dtype: H={H} N={N} C={C} as {args.dtype} does not fit one GPU: "
                         f"{need / 1e9:.1f} GB of slab, U and ensemble sums, {have / 1e9:.1f} GB on the device")

    t = time.time()
    ds = SyntheticDataset(H, N, C, seed=args.seed, device=dev, dtype=dt)
    labels_dev, labels_host = ds.labels.to(dev), ds.labels_host.numpy()
    torch.cuda.synchronize()
    t_gen = time.time() - t

    def make(preds):
        random.seed(0)
        t = time.time()
        sel = CODA(TensorDataset(preds, ds.labels, n_offset=0, n_global=N))
        torch.cuda.synchronize()
        return sel, time.time() - t

    sel, t_init = make(ds.preds)
    eng = sel.engine
    sel.run_steps(max(2, args.warmup), labels_dev)        # the first step is eager, then the capture
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    sel.run_steps(args.steps, labels_dev)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    eng.check_flags(sync=True)
    hist = sel.history()
    out = {"picks": np.asarray(hist[0])[-args.steps:], "eig": sel.eig.cpu().numpy(),
           "pbest": sel.get_pbest().cpu().numpy()}

    eng.loop_prepare(labels_dev)
    torch.cuda.synchronize()
    eng.start_profile(["coda_b200_pi_rank1"])
    for _ in range(5):
        eng.loop_eager()
    prof = eng.stop_profile().get("coda_b200_pi_rank1")
    r1_ms = prof[1] / max(1, prof[0]) if prof else None

    def api_step():
        idx, q = sel.get_next_item_to_label()
        sel.add_label(idx, int(labels_host[idx]), q)
        return int(sel.get_best_model_prediction())
    for _ in range(5):
        api_step()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(args.e2e_steps):
        api_step()
    torch.cuda.synchronize()
    ms_e2e = (time.perf_counter() - t) * 1e3 / args.e2e_steps
    shadow = eng.n_shadow
    sel.close()
    del sel, eng

    identical = None
    if args.compare_widened:
        torch.cuda.empty_cache()
        sel, _ = make(ds.preds.float())
        sel.run_steps(max(2, args.warmup), labels_dev)
        sel.run_steps(args.steps, labels_dev)
        torch.cuda.synchronize()
        h = sel.history()
        w = {"picks": np.asarray(h[0])[-args.steps:], "eig": sel.eig.cpu().numpy(), "pbest": sel.get_pbest().cpu().numpy()}
        identical = {k: bool(np.array_equal(out[k].view(np.uint8), w[k].view(np.uint8))) for k in out}
        sel.close()

    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in out.items():
            np.save(os.path.join(args.dump_outputs, k + ".npy"), v)
    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip() or None
    except Exception:
        card = None
    line = {"metric": "acquisition steps/sec by slab dtype", "dtype": args.dtype, "value": args.steps / (ms / 1e3),
            "unit": "steps/s", "ms_per_step": ms / args.steps, "steps": args.steps, "warmup": args.warmup,
            "e2e": {"value": 1e3 / ms_e2e, "ms_per_step": ms_e2e, "steps": args.e2e_steps},
            "gen_s": t_gen, "init_s": t_init, "shadow_models": shadow, "k_pi_rank1_ms": r1_ms,
            "slab_GB": H * N * C * dt.itemsize / 1e9, "workload": dict(H=H, N=N, C=C, seed=args.seed),
            "identical_to_fp32_widening": identical, "card": card,
            "loop": "value: CUDA graph, one replay per step; e2e: public API, host oracle (main.py:91-94)"}
    sys.stdout.flush()
    os.write(real_stdout, (json.dumps(line) + "\n").encode())


if __name__ == "__main__":
    main()
