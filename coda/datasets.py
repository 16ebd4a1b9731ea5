import os

from coda_b200.datasets import Dataset as _Dataset
from coda_b200.datasets import load_route


class Dataset(_Dataset):
    """reference coda/datasets.py, loaded the way ``coda_b200.datasets.load_route`` decides from the ``CODA_B200_*``
    settings.  ``CODA_B200_KEEP_DTYPE=1`` keeps a stored fp16 / bf16 slab at its width (half the device memory, the same
    results as the fp32 widening).  ``CODA_B200_SHARD_LOAD=1``, or a slab larger than the target device's free memory
    with more than one GPU visible, loads it as N-range pieces over the GPUs (``coda_b200.datasets.ShardedSlab``;
    ``CODA_B200_GPUS`` pieces, else one per visible GPU).

    A file written by ``coda_b200.CompactSlab.save`` loads as a compact slab, and ``CODA_B200_COMPACT_K=K`` compacts a
    dense task file to its top-K form as it loads (opt-in: the compact form approximates the tail classes, so results
    differ from the dense run).  The piece count follows the same rule on the compact byte count
    (``coda_b200.datasets.ShardedCompactSlab`` for more than one piece).

    ``CODA_B200_HOST_SLAB=1``, or a dense slab larger than the target device's free memory with exactly one GPU
    visible, keeps it in host memory (``coda_b200.datasets.HostSlab``) and runs it exactly on that GPU;
    ``CODA_B200_HOST_SLAB=0`` never does.  With more than one GPU visible and neither ``CODA_B200_HOST_SLAB`` nor
    ``CODA_B200_SHARD_LOAD`` set, a dense slab larger than the summed free memory of the GPUs its pieces would use stays
    in host memory as N-range pieces, one per GPU (``coda_b200.datasets.ShardedHostSlab``; ``CODA_B200_GPUS`` pieces,
    else one per visible GPU).  Compact files and ``CODA_B200_COMPACT_K`` take precedence."""

    def __init__(self, filepath, device):
        super().__init__(filepath, device, **load_route(filepath, device, os.environ))
