"""Host side of 16-bit prediction slabs: the synthetic generator's dtype, the loaders' keep_dtype, shadow sizing with
2-byte model slots and the slab-format codes.  No GPU needed."""
import pytest
import torch

from coda_b200 import _native as nat
from coda_b200.datasets import Dataset, ShardedFileDataset
from coda_b200.engine import shadow_slots
from coda_b200.synth import synth

GB = 1 << 30


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("dense", [False, True])
def test_synth_dtype_is_the_rounded_fp32_slab(dt, dense):
    H, N, C = 5, 70_000, 7                       # two generator blocks
    ref, lab = synth(H, N, C, seed=3, dense=dense)
    x, lab16 = synth(H, N, C, seed=3, dense=dense, dtype=dt)
    assert x.dtype == dt and torch.equal(lab, lab16)
    assert torch.equal(x.view(torch.int16), ref.to(dt).view(torch.int16))
    lo, hi = 65_000, 66_000                      # straddles the block boundary
    part, _ = synth(H, N, C, seed=3, dense=dense, n_lo=lo, n_hi=hi, dtype=dt)
    assert torch.equal(part.view(torch.int16), x[:, lo:hi].view(torch.int16))


def _save(tmp_path, t):
    f = str(tmp_path / "task.pt")
    torch.save(t, f)
    return f


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16, torch.float32, torch.float64])
def test_keep_dtype_loaders(tmp_path, dt):
    x, _ = synth(4, 301, 6, seed=1)
    x = x.to(dt)
    f = _save(tmp_path, x)
    kept = dt if dt in (torch.float16, torch.bfloat16, torch.float32) else torch.float32
    d0 = Dataset(f, "cpu")
    d1 = Dataset(f, "cpu", keep_dtype=True)
    assert d0.preds.dtype == torch.float32 and torch.equal(d0.preds, x.float())
    assert d1.preds.dtype == kept and torch.equal(d1.preds, x.to(kept))
    for rank in range(3):
        s0 = ShardedFileDataset(f, "cpu", rank=rank, world=3)
        s1 = ShardedFileDataset(f, "cpu", rank=rank, world=3, keep_dtype=True)
        lo = s0.n_offset
        n = s0.preds.shape[1]
        assert s1.n_offset == lo and s1.preds.dtype == kept
        assert torch.equal(s0.preds, x[:, lo:lo + n].float())
        assert torch.equal(s1.preds, x[:, lo:lo + n].to(kept))


def test_shim_keep_dtype_knob(tmp_path, monkeypatch):
    import coda.datasets
    x, _ = synth(3, 50, 4, seed=2, dtype=torch.float16)
    f = _save(tmp_path, x)
    monkeypatch.delenv("CODA_B200_KEEP_DTYPE", raising=False)
    assert coda.datasets.Dataset(f, "cpu").preds.dtype == torch.float32
    monkeypatch.setenv("CODA_B200_KEEP_DTYPE", "1")
    assert coda.datasets.Dataset(f, "cpu").preds.dtype == torch.float16


def test_shadow_slots_with_two_byte_model_slots():
    N, C = 500_000, 100
    cs = (N + 7) // 8 * 8
    s16, s32 = cs * C * 2, cs * C * 4
    free, reserve = 20 * GB, 4 * N * C + GB
    S, ne = shadow_slots(free, reserve, s16, want=256, ens=True, ens_slot_bytes=s32)
    assert ne == 1 and S == (free - reserve - s32) // s16
    S32, _ = shadow_slots(free, reserve, s32, want=256, ens=True)
    assert S >= 2 * S32
    # the fp32 ensemble slot does not fit, a 2-byte model slot does
    assert shadow_slots(reserve + s32 - 1, reserve, s16, want=256, ens=True, ens_slot_bytes=s32) == (1, 0)
    assert shadow_slots(reserve + s32, reserve, s16, want=256, ens=True, ens_slot_bytes=s32) == (0, 1)
    assert shadow_slots(reserve + s16, reserve, s16, want=256, ens=False, ens_slot_bytes=s32) == (1, 0)
    # without ens_slot_bytes every slot is sized alike (the fp32 behaviour)
    assert shadow_slots(free, reserve, s32, want=256, ens=True) == shadow_slots(free, reserve, s32, 256, True,
                                                                                ens_slot_bytes=s32)


def test_slab_format_codes():
    assert nat.slab_format(torch.float32) == nat.SLAB_F32 == 0
    assert nat.slab_format(torch.float16) == nat.SLAB_F16 == 1
    assert nat.slab_format(torch.bfloat16) == nat.SLAB_BF16 == 2
    for dt in (torch.float64, torch.int32, torch.float8_e4m3fn):
        with pytest.raises(TypeError):
            nat.slab_format(dt)
