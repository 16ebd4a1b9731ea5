"""``from coda.baselines.modelpicker import TASK_EPS`` (main.py:73).

The reference tunes ModelPicker's epsilon per task; that table is not shipped here, so every task falls back to
main.py's default (epsilon = 0.46, with main.py's "not in TASK_EPS; using default" line).  Pass a tuned value with
``ModelPicker(dataset, epsilon=...)``.  With ``CODA_REFERENCE_PATH`` set, ``coda.baselines`` has already put the
reference's own module under this name."""
from coda_b200.baselines import ModelPicker  # noqa: F401

TASK_EPS = {}
