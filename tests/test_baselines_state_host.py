"""Host side of the competing selectors' checkpoints: ``pack_state`` builds a state from plain host values, and
``check_state`` refuses a state of another method, task shape, epsilon or version before anything is touched."""
import io
import random

import numpy as np
import pytest
import torch

from coda_b200.baselines import STATE_FIELDS, STATE_VERSION, check_state, pack_state

H, N, C = 5, 40, 3


def _fields(method, M=3):
    if method in ("iid", "uncertainty"):
        return {"risk_sum": torch.tensor([1.0, 0.0, 2.0, 3.0, 1.0])}
    if method in ("activetesting", "vma"):
        return {"losses": (torch.arange(M * H).reshape(M, H) % 2).float(), "qs": [0.25, 0.125, 1 / 3], "M": M}
    return {"posterior": torch.full((H,), 0.2), "correct_counts": torch.tensor([3, 1, 0, 2, 3]), "n_disagree": 17}


def _state(method, epsilon=None):
    random.seed(4)
    torch.manual_seed(4)
    hist = {"idx": np.array([7, 2], np.int64), "q": np.array([0.25, 1 / 3]), "tie": np.array([0, 1], np.int32),
            "best": np.array([4, 0], np.int32), "best_tie": np.array([1, 0], np.int32)}
    return pack_state(method, H, N, C, epsilon, labeled=[11, 7, 2], labels=[0, 2, 1], removed=[30, 5],
                      stochastic=True, history=hist, fields=_fields(method),
                      rng={"python": random.getstate(), "torch": torch.get_rng_state(),
                           "cuda": torch.zeros(16, dtype=torch.uint8)})


def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=True)


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b)
    if isinstance(a, dict):
        return isinstance(b, dict) and a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return type(a) is type(b) and len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return type(a) is type(b) and a == b


@pytest.mark.parametrize("method", sorted(STATE_FIELDS))
def test_packed_state_survives_a_weights_only_round_trip(method):
    eps = 0.3 if method == "model_picker" else None
    sd = _state(method, eps)
    assert sd["version"] == STATE_VERSION and sd["method"] == method and (sd["H"], sd["N"], sd["C"]) == (H, N, C)
    assert sd["removed"] == [5, 30] and sd["dev_steps"] == 2
    assert [sd["history"][k].dtype for k in ("idx", "q", "tie", "best", "best_tie")] == [
        torch.int64, torch.float64, torch.int32, torch.int32, torch.int32]
    back = _roundtrip(sd)
    assert _same(sd, back)
    check_state(back, method, H, N, C, eps)
    random.seed(99)
    random.setstate(back["rng"]["python"])               # the tuple form random.setstate takes
    torch.set_rng_state(back["rng"]["torch"])
    assert random.random() == (random.seed(4), random.random())[1]


def test_an_empty_state_packs_and_checks():
    sd = _roundtrip(pack_state("iid", H, N, C, fields={"risk_sum": torch.zeros(H)}))
    check_state(sd, "iid", H, N, C)
    assert sd["dev_steps"] == 0 and all(v.numel() == 0 for v in sd["history"].values())


def test_the_validator_refuses_another_method_shape_epsilon_and_version():
    sd = _state("model_picker", 0.46)
    check_state(sd, "model_picker", H, N, C, 0.46)
    with pytest.raises(ValueError, match="method"):
        check_state(sd, "iid", H, N, C)
    with pytest.raises(ValueError, match="method"):
        check_state(_state("activetesting"), "vma", H, N, C)
    for shape in ((H + 1, N, C), (H, N - 1, C), (H, N, C + 1)):
        with pytest.raises(ValueError, match="task"):
            check_state(sd, "model_picker", *shape, 0.46)
    with pytest.raises(ValueError, match="epsilon"):
        check_state(sd, "model_picker", H, N, C, 0.3)
    with pytest.raises(ValueError, match="epsilon"):
        check_state(_state("iid"), "iid", H, N, C, 0.46)
    for v in (0, 2, None):
        with pytest.raises(ValueError, match="version"):
            check_state(dict(sd, version=v), "model_picker", H, N, C, 0.46)
    with pytest.raises(ValueError):
        check_state([sd], "model_picker", H, N, C, 0.46)


def test_the_validator_refuses_states_that_do_not_fit_the_task():
    sd = _state("vma")
    bad = [dict(sd, d_l_ys=[0, 2]), dict(sd, removed=[5, 7]), dict(sd, removed=[N]), dict(sd, dev_steps=3),
           dict(sd, fields=dict(sd["fields"], qs=[0.5])), dict(sd, fields=dict(sd["fields"], losses=torch.zeros(3, H + 1))),
           {k: v for k, v in sd.items() if k != "rng"}, dict(sd, fields={"losses": sd["fields"]["losses"]})]
    for b in bad:
        with pytest.raises(ValueError):
            check_state(b, "vma", H, N, C)
    mp = _state("model_picker", 0.46)
    with pytest.raises(ValueError, match="sums"):
        check_state(dict(mp, fields=dict(mp["fields"], posterior=torch.ones(H - 1))), "model_picker", H, N, C, 0.46)
