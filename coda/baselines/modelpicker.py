"""``from coda.baselines.modelpicker import TASK_EPS`` (main.py:73).

The reference tunes ModelPicker's epsilon per task; that table is not shipped here, so by default every task falls back
to main.py's default (epsilon = 0.46, with main.py's "not in TASK_EPS; using default" line).  ``python -m
coda_b200.eps_search`` searches a task's epsilon on the GPU and writes ``best_epsilons.json``; with
``CODA_B200_TASK_EPS`` naming such a file, ``TASK_EPS[task]`` is its ``best_avg`` for every task in it.  Or pass a value
with ``ModelPicker(dataset, epsilon=...)``.  With ``CODA_REFERENCE_PATH`` set, ``coda.baselines`` has already put the
reference's own module under this name."""
import json
import os

from coda_b200.baselines import ModelPicker  # noqa: F401

TASK_EPS = {}

if os.environ.get("CODA_B200_TASK_EPS"):
    with open(os.environ["CODA_B200_TASK_EPS"]) as _f:
        for _task, _v in json.load(_f).items():     # a --pred-dir search keys by file name: <task>.pt
            TASK_EPS[_task[:-3] if _task.endswith(".pt") else _task] = float(_v["best_avg"])
