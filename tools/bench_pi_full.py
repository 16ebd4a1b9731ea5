"""Time coda_b200_pi_full (fp32 SIMT) against coda_b200_pi_full_tc (wgmma) on a synthetic slab: python tools/bench_pi_full.py [H N C]."""
import sys

import torch

sys.path.insert(0, ".")
from coda_b200 import _native as nat  # noqa: E402


def main():
    H, N, C = (int(x) for x in sys.argv[1:4]) if len(sys.argv) >= 4 else (256, 131072, 100)
    lib = nat.load()
    nat.require_device()
    dev = torch.device("cuda:0")
    preds = torch.rand((H, N, C), device=dev)
    preds /= preds.sum(-1, keepdim=True)
    D = 0.2 + 2 * torch.rand((H, C, C), device=dev)
    st = torch.cuda.current_stream().cuda_stream
    scratch = torch.empty(int(lib.coda_b200_pi_full_tc_scratch_bytes(H, C)), dtype=torch.uint8, device=dev)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    U1, U2 = torch.empty((N, C), device=dev), torch.empty((N, C), device=dev)

    def run(name, fn, reps):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        gb = H * N * C * 4 / 1e9
        print(f"{name}: {ms:.3f} ms  slab {gb:.1f} GB -> {gb / ms:.2f} TB/s  {2 * H * N * C * C / ms / 1e9:.1f} TFLOP/s (fp32-equivalent)", flush=True)
        return ms
    import os
    ref = torch.einsum("hns,hcs->nc", preds[:, :2048].double(), D.double())
    for g in os.environ.get("PI_DRAIN_SWEEP", "2").split(","):
        os.environ["CODA_B200_PI_DRAIN"] = g
        run(f"tc  drain={g}", lambda: nat.check(lib.coda_b200_pi_full_tc(preds.data_ptr(), N * C, D.data_ptr(), H, N, C, U2.data_ptr(),
                                                                          scratch.data_ptr(), flags.data_ptr(), st)), 5)
        u = U2[:2048].double()
        raw = ((u - ref).abs() / ref).max().item()
        nrm = ((u / u.sum(1, keepdim=True) - ref / ref.sum(1, keepdim=True)).abs() / (ref / ref.sum(1, keepdim=True))).max().item()
        print(f"   vs fp64: raw {raw:.2e}  row-normalised {nrm:.2e}", flush=True)
    run("tc  ", lambda: nat.check(lib.coda_b200_pi_full_tc(preds.data_ptr(), N * C, D.data_ptr(), H, N, C, U2.data_ptr(),
                                                            scratch.data_ptr(), flags.data_ptr(), st)), 5)
    print("flags", hex(int(flags.item())))
    run("simt", lambda: nat.check(lib.coda_b200_pi_full(preds.data_ptr(), N * C, D.data_ptr(), H, N, C, U1.data_ptr(), st)), 2)
    rel = ((U2 - U1).abs() / U1).max().item()
    print("max rel diff tc vs simt", rel)
    u = U1[:2048].double()
    print("simt vs fp64: raw %.2e  row-normalised %.2e" % (((u - ref).abs() / ref).max().item(),
          ((u / u.sum(1, keepdim=True) - ref / ref.sum(1, keepdim=True)).abs() / (ref / ref.sum(1, keepdim=True))).max().item()))


if __name__ == "__main__":
    main()
