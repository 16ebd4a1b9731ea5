"""The majority shortcut's base E[n][t'] travels as the first ordinary term of the rank-1 gather list, read from the
class-major ensemble slot of the shadow or from the item-major ensemble sums; and the shadow is sized so that shards
sharing a device split the spare memory.  Sizing arithmetic runs on the CPU, the refresh on the GPU."""
import pytest
import torch

from coda_b200.engine import shadow_slots

GB = 1 << 30


def test_shadow_slots_keep_every_reserve_and_split_the_rest():
    slot = 200 * 10 ** 6
    for k in (1, 2, 3, 4):
        free, reserve, shares = 28 * GB, GB + 4 * 10 ** 8, []
        for i in range(k):
            S, ne = shadow_slots(free, reserve, slot, want=256, ens=True, left=k - i, total=k)
            assert ne == 1
            shares.append(S + ne)
            free -= (S + ne) * slot
        assert free >= k * reserve, (k, free)
        assert max(shares) - min(shares) <= 1, shares
        assert free - k * reserve < k * slot            # nothing worth a slot is left unused
    assert shadow_slots(28 * GB, GB, slot, want=256, ens=True) == (143, 1)
    assert shadow_slots(28 * GB, GB, slot, want=3, ens=True) == (3, 1)
    assert shadow_slots(28 * GB, GB, slot, want=0, ens=True) == (0, 1)
    assert shadow_slots(28 * GB, GB, slot, want=256, ens=False) == (144, 0)
    assert shadow_slots(GB + slot - 1, GB, slot, want=256, ens=True) == (0, 0)
    assert shadow_slots(GB + slot, GB, slot, want=256, ens=True) == (0, 1)
    assert shadow_slots(GB // 2, GB, slot, want=256, ens=True) == (0, 0)


def _terms(eng):
    a = eng.terms.cpu()
    nt, tp = int(a[0]), int(a[1])
    return nt, tp, a[2:2 + 4 * nt].view(nt, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(64, 20000, 20, 5), (37, 3001, 7, 11)])
def test_ensemble_term_source_leaves_the_bits_alone(shape, monkeypatch):
    """Shadow off (E from the item-major sums, every model from the slab), the ensemble slot only, three model slots
    plus the ensemble slot, and every model in the shadow: the same U, column sums, pi_hat and picks after every
    label."""
    from coda_b200 import CODA, TensorDataset
    from coda_b200.synth import synth
    H, N, C, seed = shape
    preds, labels = synth(H, N, C, seed=seed)
    dev = torch.device("cuda:0")
    preds, labels = preds.to(dev), labels.to(dev)
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    envs = {"off": {"CODA_B200_SHADOW": "0"}, "ens_only": {"CODA_B200_SHADOW_MODELS": "0"},
            "three": {"CODA_B200_SHADOW_MODELS": "3"}, "all": {}}
    sels = {}
    for name, env in envs.items():
        for k in ("CODA_B200_SHADOW", "CODA_B200_SHADOW_MODELS"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        sels[name] = CODA(TensorDataset(preds, labels))
    for k in ("CODA_B200_SHADOW", "CODA_B200_SHADOW_MODELS"):
        monkeypatch.delenv(k, raising=False)
    assert sels["off"].engine.shadow is None
    assert sels["ens_only"].engine.n_shadow == 0 and sels["ens_only"].engine.shadow.shape[0] == 1
    assert sels["three"].engine.n_shadow == 3 and sels["all"].engine.n_shadow == H
    shortcut = 0
    for step, i in enumerate([3, N // 2, N - 1, 17, N // 3, 5, N // 5]):
        for s in sels.values():
            s.add_label(i, int(labels[i]), 0.0)
        torch.cuda.synchronize()
        ref = sels["off"]
        for name, s in sels.items():
            assert torch.equal(ref.engine.U, s.engine.U), (shape, step, name)
            assert torch.equal(ref.engine.pisum, s.engine.pisum) and torch.equal(ref.pi_hat, s.pi_hat), (shape, step, name)
        nt, tp, tl = _terms(sels["ens_only"].engine)
        if tp >= 0:                                     # the shortcut is on: E first, then two terms per dissenting model
            shortcut += 1
            assert nt % 2 == 1
            assert int(tl[0, 3]) == 1 and tl[0:1, 2].view(torch.float32).item() == 1.0
            nt_off, tp_off, tl_off = _terms(sels["off"].engine)
            assert (nt_off, tp_off) == (nt, tp) and int(tl_off[0, 3]) == C
            assert (tl[1:, 3] == C).all() and (_terms(sels["all"].engine)[2][:, 3] == 1).all()
    assert shortcut > 0
    picks = {name: s.get_next_item_to_label() for name, s in sels.items()}
    assert len(set(picks.values())) == 1, picks
    for s in sels.values():
        s.close()


@pytest.mark.gpu
def test_shards_on_one_device_share_the_shadow():
    """In-process shards on one GPU: every shard keeps its row cache and gets a shadow with the ensemble slot."""
    from coda_b200 import CODA, TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(32, 3000, 10, seed=6)
    dev = torch.device("cuda:0")
    sel = CODA(TensorDataset(preds.to(dev), labels.to(dev)), shards=3)
    for e in sel.engines:
        assert e.mode == "incremental" and e.ph_cache is not None
        assert e.shadow is not None and e.shadow.shape[0] == e.n_shadow + 1 and e.n_shadow == 32
    sel.close()
