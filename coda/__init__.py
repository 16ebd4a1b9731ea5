"""Drop-in ``coda`` package: the names the reference's drivers import (coda/__init__.py:1-3),
served by ``coda_b200``.  Put this repository before the reference on PYTHONPATH and
``main.py --method coda`` runs on the sm_90a kernels unchanged (see INTEGRATION.md)."""
from coda_b200.selector import CODA
from .datasets import Dataset          # the shim (CODA_B200_KEEP_DTYPE, CODA_B200_SHARD_LOAD), as coda/__init__.py:2
from coda_b200.oracle import Oracle

__all__ = ["CODA", "Dataset", "Oracle"]
