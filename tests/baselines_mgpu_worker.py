"""torchrun worker: the competing selectors with one process per GPU vs a single-GPU run of the same task (used by
test_baselines_sharded.py).
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/baselines_mgpu_worker.py
"""
import hashlib
import json
import os
import random
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from coda.options import LOSS_FNS  # noqa: E402
from coda_b200 import IID, VMA, ActiveTesting, ModelPicker, SyntheticDataset, Uncertainty  # noqa: E402
from coda_b200.dist import LocalComm, TorchComm  # noqa: E402

CLASSES = {"iid": IID, "uncertainty": Uncertainty, "activetesting": ActiveTesting, "vma": VMA, "model_picker": ModelPicker}


def _digest(b):
    return int.from_bytes(hashlib.sha256(b).digest()[:8], "little", signed=True)


def _run(ds, method, comm, labels, steps):
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)
    cls = CLASSES[method]
    sel = cls(ds, comm=comm) if method == "model_picker" else cls(ds, LOSS_FNS["acc"], comm=comm)
    out = [[int(sel.get_best_model_prediction())]]
    for _ in range(steps):
        idx, q = sel.get_next_item_to_label()
        sel.add_label(idx, int(labels[idx]), q)
        out.append([idx, q, int(sel.get_best_model_prediction()), _digest(repr(random.getstate()).encode()),
                    _digest(torch.get_rng_state().numpy().tobytes()),
                    _digest(torch.cuda.get_rng_state().numpy().tobytes())])
    sel.close()
    return out


def main():
    rank, world, lr = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(lr)
    dev = torch.device("cuda", lr)
    dist.init_process_group("nccl", device_id=dev)
    H, N, C, steps = 48, 30011, 14, 12
    res = {}
    for method in CLASSES:
        ds = SyntheticDataset(H, N, C, seed=4, device=dev, rank=rank, world=world)
        trace = _run(ds, method, TorchComm(), ds.labels_host, steps)
        allt = [None] * world
        dist.all_gather_object(allt, trace)
        res[method] = {"trace": trace, "same_on_all_ranks": all(t == trace for t in allt)}
        if rank == 0:
            full = SyntheticDataset(H, N, C, seed=4, device=dev)
            res[method]["trace_single"] = _run(full, method, LocalComm(), full.labels_host, steps)
            del full
        del ds
        dist.barrier()
    if rank == 0:
        print("BASELINES_MGPU " + json.dumps(res), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
