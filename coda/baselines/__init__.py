"""The competing selectors (IID, Uncertainty, ActiveTesting, VMA, ModelPicker) that ``main.py --method ...`` runs next
to CODA (main.py:10, 67-80).  Resolution order:

1. ``CODA_REFERENCE_PATH`` names a reference checkout whose ``coda/baselines/<name>.py`` modules load: the reference's
   own classes, unchanged (they also take ``coda.baselines.<name>`` in ``sys.modules``, so
   ``from coda.baselines.modelpicker import TASK_EPS`` then gets the reference's table);
2. otherwise the GPU classes of ``coda_b200.baselines`` (one sm_90a device, dense slab; a CPU ``dataset.preds`` raises
   ``NotImplementedError``)."""
import importlib.util
import os
import sys

_NAMES = {"IID": "iid", "ActiveTesting": "activetesting", "VMA": "vma", "ModelPicker": "modelpicker",
          "Uncertainty": "uncertainty"}


def _load_reference(path):
    out = {}
    base = os.path.join(path, "coda", "baselines")
    for cls, mod in _NAMES.items():
        f = os.path.join(base, mod + ".py")
        if not os.path.exists(f):
            return None
        spec = importlib.util.spec_from_file_location(f"coda.baselines.{mod}", f)
        m = importlib.util.module_from_spec(spec)
        sys.modules[spec.name] = m
        spec.loader.exec_module(m)
        out[cls] = getattr(m, cls)
    return out


_ref = os.environ.get("CODA_REFERENCE_PATH")
_loaded = None
if _ref and os.path.isdir(_ref):
    try:
        _loaded = _load_reference(_ref)
    except Exception:  # pragma: no cover - the reference needs matplotlib etc.
        _loaded = None
if _loaded is None:
    from coda_b200 import baselines as _ours
    _loaded = {cls: getattr(_ours, cls) for cls in _NAMES}
for _cls in _NAMES:
    globals()[_cls] = _loaded[_cls]
