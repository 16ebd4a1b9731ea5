"""A slab loaded as N-range pieces (``ShardedSlab``) on the GPU: the loader against ``torch.load``, the true-loss kernel
against torch's arg-max, ``Oracle.true_losses`` bit for bit against the single-tensor path, CODA and the five competing
selectors on pieces against ``shards=k`` on one tensor, and main.py's cfg1 driver loading sharded.  Everything runs on
one GPU with the pieces sharing it; the multi-device case skips below 2 GPUs."""
import ctypes as ct
import os
import random

import numpy as np
import pytest
import torch

from helpers import golden_slab, load_golden

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _save(tmp_path, t, name="task.pt"):
    p = str(tmp_path / name)
    torch.save(t, p)
    return p


# ------------------------------------------------------------------------------------------------------------------
# loader
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("shards", [1, 2, 3, 4])
def test_every_piece_equals_torch_load(tmp_path, dtype, keep, shards):
    from coda_b200.datasets import Dataset, ShardedSlab
    from coda_b200.synth import shard_range
    H, N, C = 5, 1003, 7                                     # N not divisible by 2, 3 or 4
    t = torch.rand(H, N, C, generator=torch.Generator().manual_seed(shards)).to(dtype)
    p = _save(tmp_path, t)
    torch.save(torch.randint(0, C, (N,)), p.replace(".pt", "_labels.pt"))
    for chunk in (1 << 20, 6 * t.element_size(), 50 * t.element_size()):   # 6 and 50 elements split every model's range
        ds = Dataset(p, DEV, keep_dtype=keep, shards=shards, gpus=1, chunk_bytes=chunk)
        s = ds.preds
        assert isinstance(s, ShardedSlab) and len(s.pieces) == shards and s.shape == t.shape
        want = torch.load(p)
        want = want if keep else want.float()
        assert s.dtype == want.dtype
        for r, piece in enumerate(s.pieces):
            lo, hi = shard_range(N, r, shards)
            assert s.offsets[r] == lo and piece.device == DEV and piece.is_contiguous()
            assert torch.equal(piece.cpu().view(torch.uint8), want[:, lo:hi].contiguous().view(torch.uint8))
        assert ds.labels.device == DEV and torch.equal(ds.labels.cpu(), torch.load(p.replace(".pt", "_labels.pt")))


@pytest.mark.parametrize("dtype,keep", [(torch.float32, False), (torch.float16, False), (torch.bfloat16, True)])
def test_load_holds_no_more_than_the_pieces_and_one_chunk(tmp_path, dtype, keep):
    from coda_b200.datasets import load_sharded
    H, N, C = 16, 20011, 10
    p = _save(tmp_path, torch.rand(H, N, C).to(dtype))
    chunk = 3 << 16
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    s = load_sharded(p, DEV, keep, shards=3, gpus=1, chunk_bytes=chunk)
    peak = torch.cuda.max_memory_allocated(DEV) - base
    pieces = sum(x.numel() * x.element_size() for x in s.pieces)
    slack = 512 * (len(s.pieces) + 1)                         # the caching allocator's 512-byte rounding
    assert peak <= pieces + (0 if keep or dtype == torch.float32 else chunk) + slack, (peak, pieces)


def test_shim_loads_sharded_on_opt_in(tmp_path, monkeypatch, capsys):
    from coda import Dataset
    from coda_b200.datasets import ShardedSlab
    t = torch.rand(3, 100, 4)
    p = _save(tmp_path, t)
    monkeypatch.setenv("CODA_B200_SHARD_LOAD", "1")
    monkeypatch.setenv("CODA_B200_GPUS", "3")
    ds = Dataset(p, DEV)
    assert isinstance(ds.preds, ShardedSlab) and len(ds.preds.pieces) == 3
    assert "Loaded preds of shape torch.Size([3, 100, 4])" in capsys.readouterr().out
    monkeypatch.delenv("CODA_B200_SHARD_LOAD")
    assert isinstance(Dataset(p, DEV).preds, torch.Tensor)   # a slab that fits loads as today


# ------------------------------------------------------------------------------------------------------------------
# true-loss kernel
# ------------------------------------------------------------------------------------------------------------------
def _counts(preds_view, labels, H, N, C, model_stride):
    from coda_b200 import _native as nat
    out = torch.full((H,), -7, dtype=torch.int64, device=DEV)       # poisoned: the entry point must zero it
    nat.call("coda_b200_true_loss_counts", ct.c_void_p(preds_view.data_ptr()), nat.slab_format(preds_view.dtype),
             model_stride, H, N, C, ct.c_void_p(labels.data_ptr()), ct.c_void_p(out.data_ptr()), None)
    torch.cuda.synchronize()
    return out.cpu()


def _torch_counts(x, labels):
    return (torch.argmax(x, dim=-1) == labels[None, :]).sum(1).cpu()


def _nasty(H, N, C, dtype, seed):
    """Scores with exact ties, NaN, +-0 and out-of-range labels."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.rand(H, N, C, device=DEV, generator=g)
    x = (x * 4).floor() / 4                                  # many exact ties
    if N > 3:
        x[:, 1] = 0.0
        x[:, 2] = -0.0
        x[:, 3, C // 2:] = -0.0
    if N > 8 and C > 1:
        x[0, 5, C - 1] = float("nan")
        x[-1, 6, :] = float("nan")
        x[:, 7, 0] = float("nan")
    labels = torch.randint(0, C, (N,), device=DEV, generator=g)
    if N > 10:
        labels[9] = C
        labels[10] = -1
    return x.to(dtype), labels


@pytest.mark.parametrize("C", [1, 2, 3, 10, 100, 1000, 4096])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_true_loss_counts_equal_torch_argmax(C, dtype):
    for H, N in [(1, 1), (3, 17), (7, 301), (2, 5003)]:
        if C >= 1000 and N > 301:
            N = 97
        x, labels = _nasty(H, N, C, dtype, seed=C * 31 + N)
        got = _counts(x, labels, H, N, C, N * C)
        assert torch.equal(got, _torch_counts(x, labels)), (H, N, C)


@pytest.mark.parametrize("C", [3, 10, 100])
def test_true_loss_counts_on_n_range_views(C):
    H, N = 11, 2001
    x, labels = _nasty(H, N, C, torch.float32, seed=C)
    for lo, hi in [(0, 1), (1, 2), (3, 700), (699, 2001), (1333, 1337)]:
        v = x[:, lo:hi]
        got = _counts(v, labels[lo:hi], H, hi - lo, C, N * C)
        assert torch.equal(got, _torch_counts(v, labels[lo:hi])), (lo, hi)


def test_true_loss_counts_at_1024_models():
    for C in (2, 100):
        x, labels = _nasty(1024, 129, C, torch.float16, seed=C)
        assert torch.equal(_counts(x, labels, 1024, 129, C, 129 * C), _torch_counts(x, labels))


@pytest.mark.parametrize("N", [1, 2, 3, 7, 100, 1000, 4097, 65537, 333331, 1048576, 999983])
def test_oracle_true_losses_on_pieces_are_torchs_bits(N):
    from coda.options import LOSS_FNS
    from coda_b200 import Oracle, TensorDataset
    from coda_b200.datasets import ShardedSlab
    from coda_b200.synth import shard_range
    H, C = (7, 3) if N < 100000 else (3, 2)
    x, labels = _nasty(H, N, C, torch.float32, seed=N)
    labels = labels.clamp(0, C - 1)
    want = Oracle(TensorDataset(x, labels), loss_fn=LOSS_FNS["acc"]).true_losses(x)
    for k in (1, 2, 3):
        k = min(k, N)
        s = ShardedSlab([x[:, slice(*shard_range(N, r, k))].contiguous() for r in range(k)])
        got = Oracle(TensorDataset(s, labels), loss_fn=LOSS_FNS["acc"]).true_losses(s)
        assert got.device == want.device and got.dtype == torch.float32
        assert got.cpu().numpy().tobytes() == want.cpu().numpy().tobytes(), (N, k)


# ------------------------------------------------------------------------------------------------------------------
# CODA on pieces
# ------------------------------------------------------------------------------------------------------------------
def _pieces_of(preds, k):
    from coda_b200.datasets import ShardedSlab
    from coda_b200.synth import shard_range
    N = preds.shape[1]
    return ShardedSlab([preds[:, slice(*shard_range(N, r, k))].contiguous().to(DEV) for r in range(k)])


def _pair(preds, labels, k, **kw):
    from coda_b200 import CODA, TensorDataset
    ref = CODA(TensorDataset(preds.to(DEV), labels.to(DEV)), shards=k, **kw)
    s = _pieces_of(preds, k)
    pcs = CODA(TensorDataset(s, labels.to(DEV)), **kw)
    assert len(pcs.engines) == k and [e.preds.data_ptr() for e in pcs.engines] == [p.data_ptr() for p in s.pieces]
    return ref, pcs


def _same_state(a, b):
    assert torch.equal(a.dirichlets, b.dirichlets) and torch.equal(a.pi_hat, b.pi_hat)
    assert torch.equal(a.get_pbest(), b.get_pbest()) and torch.equal(a.pi_hat_xi, b.pi_hat_xi)


@pytest.mark.parametrize("k", [1, 2, 3])
def test_coda_on_pieces_equals_shards_on_one_tensor_api(k):
    g = load_golden("traj_small_h32_n3000_c10")
    preds, labels = golden_slab(g)
    random.seed(0)
    ref, pcs = _pair(preds, labels, k)
    _same_state(ref, pcs)
    for step in range(int(g["steps"])):
        st = random.getstate()
        i1, q1 = ref.get_next_item_to_label()
        after = random.getstate()
        random.setstate(st)
        i2, q2 = pcs.get_next_item_to_label()
        assert (i1, q1) == (i2, q2) and random.getstate() == after and i1 == int(g["idx"][step])
        ref.add_label(i1, int(labels[i1]), q1)
        pcs.add_label(i2, int(labels[i2]), q2)
        assert int(ref.get_best_model_prediction()) == int(pcs.get_best_model_prediction())
        _same_state(ref, pcs)


def _tie_slab():
    """traj_tiny's items three times over: exact EIG ties on every step, copies on different pieces."""
    g = load_golden("traj_tiny_h8_n300_c5")
    preds, labels = golden_slab(g)
    order = torch.arange(preds.shape[1]).repeat(3)
    return preds[:, order].contiguous(), labels[order].contiguous()


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("tie_rule", ["first", "reference"])
def test_coda_run_steps_on_pieces(k, tie_rule):
    if tie_rule == "reference":
        preds, labels = _tie_slab()
    else:
        preds, labels = golden_slab(load_golden("traj_small_h32_n3000_c10"))
    random.seed(5)
    ref, pcs = _pair(preds, labels, k)
    random.seed(5)
    ref.run_steps(12, labels.to(DEV), record_best=True, tie_rule=tie_rule)
    st = random.getstate()
    random.seed(5)
    pcs.run_steps(12, labels.to(DEV), record_best=True, tie_rule=tie_rule)
    assert random.getstate() == st
    for a, b in zip(ref.history(), pcs.history()):
        assert np.asarray(a).tobytes() == np.asarray(b).tobytes()
    assert ref.best_history()[0].tolist() == pcs.best_history()[0].tolist()
    if tie_rule == "reference":
        assert sum(pcs.history()[2]) >= 3
    _same_state(ref, pcs)


def test_state_dict_crosses_layouts():
    from coda_b200 import CODA, TensorDataset
    g = load_golden("traj_small_h32_n3000_c10")
    preds, labels = golden_slab(g)
    random.seed(0)
    _, pcs = _pair(preds, labels, 3)
    for _ in range(3):
        i, q = pcs.get_next_item_to_label()
        pcs.add_label(i, int(labels[i]), q)
        pcs.get_best_model_prediction()
    sd = pcs.state_dict()
    one = CODA(TensorDataset(preds.to(DEV), labels.to(DEV)))              # pieces -> one tensor
    one.load_state_dict(sd)
    back = CODA(TensorDataset(_pieces_of(preds, 2), labels.to(DEV)))      # one tensor -> pieces
    back.load_state_dict(one.state_dict())
    for sel in (one, back):
        _same_state(pcs, sel)
    for step in range(3, int(g["steps"])):
        st = random.getstate()
        outs = []
        for sel in (pcs, one, back):
            random.setstate(st)
            i, q = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), q)
            outs.append((i, q, int(sel.get_best_model_prediction())))
        assert outs[0] == outs[1] == outs[2] and outs[0][0] == int(g["idx"][step])
        _same_state(pcs, one)
        _same_state(pcs, back)


# ------------------------------------------------------------------------------------------------------------------
# the five competing selectors on pieces
# ------------------------------------------------------------------------------------------------------------------
def _make_bl(method, ds, **kw):
    from coda.options import LOSS_FNS
    from coda_b200 import IID, VMA, ActiveTesting, ModelPicker, Uncertainty
    if method == "model_picker":
        return ModelPicker(ds, **kw)
    return {"iid": IID, "uncertainty": Uncertainty, "activetesting": ActiveTesting, "vma": VMA}[method](
        ds, LOSS_FNS["acc"], **kw)


def _seed(s=0):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)
    torch.cuda.manual_seed_all(s)


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("method", ["iid", "uncertainty", "activetesting", "vma", "model_picker"])
def test_baselines_on_pieces_equal_shards_on_one_tensor(method, k):
    from coda_b200 import TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(12, 500, 6, 3)
    lab = labels.to(DEV)
    for path in ("api", "loop"):
        runs = []
        for ds, kw in ((TensorDataset(preds.to(DEV), lab), {"shards": k}), (TensorDataset(_pieces_of(preds, k), lab), {})):
            _seed()
            sel = _make_bl(method, ds, **kw)
            assert len(sel.states) == k
            if path == "api":
                tr = [int(sel.get_best_model_prediction())]
                for _ in range(15):
                    i, q = sel.get_next_item_to_label()
                    sel.add_label(i, int(labels[i]), q)
                    tr.append((i, float(q), int(sel.get_best_model_prediction())))
            else:
                sel.run_steps(15, lab, tie_rule="reference")
                tr = [np.asarray(a).tolist() for a in list(sel.history()) + list(sel.best_history())]
            runs.append((tr, torch.get_rng_state().numpy().tobytes(), random.getstate()))
            sel.close()
        assert runs[0] == runs[1], (method, k, path)


# ------------------------------------------------------------------------------------------------------------------
# main.py, and more than one GPU
# ------------------------------------------------------------------------------------------------------------------
def test_main_py_cfg1_driver_loads_sharded(tmp_path):
    """The cfg1 driver of test_main_py_cfg1 with CODA_B200_SHARD_LOAD=1 CODA_B200_GPUS=3: three pieces on this GPU, the
    golden criteria of that file, and the same MLflow log as the unsharded run.  The driver is a fresh process under
    CUDA's default lazy module loading: the shards share this GPU and spin on each other inside the step kernels, which
    is safe only because the group loads every kernel of the library before the first exchange (csrc/preload.cu)."""
    from test_main_py_cfg1 import _compare, _run
    (tmp_path / "plain").mkdir()
    (tmp_path / "sharded").mkdir()
    g, plain, _ = _run(tmp_path / "plain")
    g, out, stdout = _run(tmp_path / "sharded", extra_env={"CODA_B200_SHARD_LOAD": "1", "CODA_B200_GPUS": "3"})
    _compare(g, out, stdout, g["iters"])
    for key in plain:
        if isinstance(plain[key], list):
            bad = [i for i, (a, b) in enumerate(zip(out[key], plain[key])) if a != b]
            assert len(out[key]) == len(plain[key]) and not bad, (key, bad[:3], [(out[key][i], plain[key][i]) for i in bad[:3]])
        if key == "params":                                   # the two runs' task files sit in different directories
            out[key].pop("data_dir"), plain[key].pop("data_dir")
        assert out[key] == plain[key], key


def test_main_py_cfg1_driver_with_three_shards_of_one_tensor(tmp_path):
    """CODA_B200_GPUS=3 without a sharded load: the tensor is split into three shards (on this GPU when it is the only
    one) in a fresh process, with lazy module loading -- the first exchange must not wait for a first-launch load."""
    from test_main_py_cfg1 import _compare, _run
    g, out, stdout = _run(tmp_path, extra_env={"CODA_B200_GPUS": "3"}, iters=20)
    _compare(g, out, stdout, 20)


def test_device_zero_holds_only_its_piece_on_several_gpus(tmp_path, monkeypatch):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    import coda_b200.dist as dist
    from coda_b200 import CODA
    from coda_b200.datasets import Dataset
    H, N, C = 64, 40000, 10
    p = _save(tmp_path, torch.rand(H, N, C).softmax(-1))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(0)
    ds = Dataset(p, DEV, gpus=n)
    pieces = ds.preds.pieces
    assert [x.device.index for x in pieces] == list(range(n))
    assert torch.cuda.memory_allocated(0) - base <= pieces[0].numel() * 4 + N * 8 + 4096     # its piece and the labels
    monkeypatch.setenv("CODA_B200_SHADOW", "0")              # no cache sized to the free memory
    monkeypatch.setattr(dist, "split_slab", lambda *a: pytest.fail("a ShardedSlab must not be re-split"))
    torch.cuda.reset_peak_memory_stats(0)
    sel = CODA(ds)
    torch.cuda.synchronize(0)
    assert [e.dev.index for e in sel.engines] == list(range(n))
    assert [e.preds.data_ptr() for e in sel.engines] == [x.data_ptr() for x in pieces]      # used in place, no copy
    # after construction device 0 holds its piece and its shard's state, never a copy of the whole slab
    assert torch.cuda.max_memory_allocated(0) - base < H * N * C * 4
