import os

from coda_b200.datasets import Dataset as _Dataset


class Dataset(_Dataset):
    """reference coda/datasets.py.  ``CODA_B200_KEEP_DTYPE=1`` keeps a stored fp16 / bf16 slab at its width (half the
    device memory, the same results as the fp32 widening)."""

    def __init__(self, filepath, device):
        super().__init__(filepath, device, keep_dtype=os.environ.get("CODA_B200_KEEP_DTYPE", "0") == "1")
