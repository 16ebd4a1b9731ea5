"""coda_b200: the CODA active-model-selection acquisition hot path on H100 (sm_90a)."""
import os as _os

# Several shards driven by one process each use their own streams and wait for each other inside kernels: give every
# stream its own hardware work queue (the default of 8 lets two streams share one, which would serialise them).
# Only effective if set before the CUDA context exists, hence at import.
_os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

from .base import ModelSelector
from .datasets import (CompactDataset, CompactSlab, Dataset, HostDataset, HostSlab, ShardedCompactSlab,
                       ShardedFileDataset, ShardedHostSlab, ShardedSlab, SyntheticCompactDataset, SyntheticDataset,
                       TensorDataset, load_compact)
from .oracle import Oracle
from .selector import CODA
from .baselines import IID, VMA, ActiveTesting, ModelPicker, Uncertainty

__all__ = ["CODA", "Dataset", "Oracle", "ModelSelector", "TensorDataset", "SyntheticDataset", "ShardedFileDataset",
           "ShardedSlab", "CompactSlab", "ShardedCompactSlab", "load_compact", "CompactDataset", "SyntheticCompactDataset",
           "HostSlab", "ShardedHostSlab", "HostDataset", "IID", "Uncertainty", "ActiveTesting", "VMA", "ModelPicker"]
