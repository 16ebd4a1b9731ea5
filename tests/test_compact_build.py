"""Building compact top-K slabs on the GPU: the compaction kernel bit for bit against its host model, the compact scan
against the dense scan, the loader against ``CompactSlab.from_dense``, the compact true losses against the dense
``Oracle.true_losses``, CODA and the five competing selectors on ``ShardedCompactSlab`` pieces against the whole slab,
the near-lossless K = C - 1 case against the dense run, and main.py's calls through the shim with
``CODA_B200_COMPACT_K``.  Everything runs on one GPU, pieces sharing it."""
import ctypes as ct
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, golden_slab, load_golden
from test_compact_build_host import compact_host

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
KS = (1, 2, 3, 4, 8)


def _build(x, K, poison=True):
    """Run coda_b200_compact_build on the CUDA (H, N, C) view ``x`` into NaN / 0xFFFF-filled outputs."""
    from coda_b200 import _native as nat
    H, N, C = x.shape
    ids = torch.full((H, N, K), -1, dtype=torch.int16, device=DEV)
    probs = torch.full((H, N, K), float("nan"), dtype=torch.float32, device=DEV)
    dropped = torch.zeros(H, dtype=torch.float32, device=DEV)
    flat = torch.zeros(H, dtype=torch.int64, device=DEV)
    flags = torch.zeros(1, dtype=torch.int32, device=DEV)
    stride = x.stride(0) if H > 1 else N * C
    nat.call("coda_b200_compact_build", ct.c_void_p(x.data_ptr()), nat.slab_format(x.dtype), stride, H, N, C, K,
             ct.c_void_p(ids.data_ptr()), ct.c_void_p(probs.data_ptr()), N * K, ct.c_void_p(dropped.data_ptr()),
             ct.c_void_p(flat.data_ptr()), ct.c_void_p(flags.data_ptr()), None)
    torch.cuda.synchronize()
    return ids.cpu(), probs.cpu(), dropped.cpu(), flat.cpu(), int(flags.item())


def _scores(H, N, C, seed, dtype=torch.float32):
    """Softmax-like rows with crafted ties (quantised rows, ties across the K-th place), uniform rows and +-0."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.rand(H, N, C, device=DEV, generator=g) ** 3
    x = x / x.sum(-1, keepdim=True)
    if N >= 8:
        x[:, 0] = 1.0 / C                                      # uniform
        x[:, 1] = (x[:, 1] * 4).floor() / 4                    # many exact ties
        x[:, 2] = 0.0
        x[:, 3] = -0.0
        x[:, 4, ::2] = -0.0
        x[:, 4, 1::2] = 0.0
        x[:, 5] = (x[:, 5] * 2).floor() / 8
        x[:, 6, : C // 2] = 0.25                               # a block of equal top scores
    return x.to(dtype)


def _same(got, x, K):
    ids, probs, dropped, flat, flags = got
    wid, wp, wd, wf = compact_host(x.float().cpu().numpy(), K)
    assert flags == 0
    assert np.array_equal(ids.numpy().astype(np.int64) & 0xFFFF, wid)
    assert probs.numpy().view(np.int32).tobytes() == wp.view(np.int32).tobytes()
    assert dropped.numpy().view(np.int32).tobytes() == wd.view(np.int32).tobytes()
    assert np.array_equal(flat.numpy(), wf)


@pytest.mark.parametrize("C", [2, 5, 10, 31, 32, 33, 100, 1000, 4096])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_kernel_equals_the_host_model(C, dtype):
    H, N = (3, 67) if C < 1000 else (2, 19)
    x = _scores(H, N, C, seed=C, dtype=dtype)
    for K in KS:
        if K < C:
            _same(_build(x, K), x, K)


@pytest.mark.parametrize("C", [5, 33, 1000])
def test_kernel_on_n_range_views(C):
    x = _scores(4, 301, C, seed=7 * C)
    for lo, hi in [(0, 1), (1, 2), (3, 150), (150, 301), (299, 301)]:
        v = x[:, lo:hi]
        for K in (1, 4):
            _same(_build(v, K), v, K)


def test_kernel_flags_bad_inputs():
    from coda_b200 import _native as nat
    for bad, flag in [(float("nan"), nat.FLAG_NONFINITE_INPUT), (float("inf"), nat.FLAG_NONFINITE_INPUT),
                      (-0.01, nat.FLAG_RANGE_INPUT), (1.001, nat.FLAG_RANGE_INPUT)]:
        x = _scores(2, 40, 10, seed=1)
        x[1, 17, 3] = bad
        assert _build(x, 4)[4] & flag, bad
    x = _scores(2, 40, 10, seed=1)
    x[0, 5, 9] = 1.0001                                        # the dense scan's tolerance
    assert _build(x, 4)[4] == 0
    x[0, 5, 9] = float("nan")
    with pytest.raises(RuntimeError, match="NaN"):
        _from_dense(x, 4)
    x[0, 5, 9] = -1.0
    with pytest.raises(ValueError, match="post-softmax"):
        _from_dense(x, 4)


def _from_dense(x, K):
    from coda_b200 import CompactSlab
    return CompactSlab.from_dense(x, K)


def test_scan_agrees_with_the_dense_scan():
    from coda_b200 import _native as nat
    for (H, N, C, dtype) in [(12, 2000, 10, torch.float32), (7, 501, 100, torch.float16), (5, 300, 1000, torch.bfloat16)]:
        x = _scores(H, N, C, seed=N, dtype=dtype)
        x[:, 10:20] = x[:1, 10:20]                              # unanimous items
        outs = []
        for compact in (None, _from_dense(x, 4)):
            hard = torch.empty(N, H, dtype=torch.int16, device=DEV)
            pseudo = torch.empty(N, dtype=torch.int32, device=DEV)
            dis = torch.empty(N, dtype=torch.uint8, device=DEV)
            flags = torch.zeros(1, dtype=torch.int32, device=DEV)
            if compact is None:
                nat.call("coda_b200_scan_slab_x", ct.c_void_p(x.data_ptr()), nat.slab_format(dtype), N * C, H, N, C,
                         ct.c_void_p(hard.data_ptr()), ct.c_void_p(pseudo.data_ptr()), ct.c_void_p(dis.data_ptr()),
                         None, ct.c_void_p(flags.data_ptr()), None)
            else:
                nat.call("coda_b200_scan_compact", ct.c_void_p(compact.ids.data_ptr()),
                         ct.c_void_p(compact.probs.data_ptr()), N * 4, H, N, C, 4, ct.c_void_p(hard.data_ptr()),
                         ct.c_void_p(pseudo.data_ptr()), ct.c_void_p(dis.data_ptr()), None,
                         ct.c_void_p(flags.data_ptr()), None)
            torch.cuda.synchronize()
            outs.append((hard.cpu(), dis.cpu()))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), (H, N, C)
        assert int(outs[0][1][10:20].sum()) == 0


# ------------------------------------------------------------------------------------------------------------------
# loader
# ------------------------------------------------------------------------------------------------------------------
def _bits(t):
    return t.cpu().contiguous().view(torch.uint8).numpy().tobytes()


def _same_slab(a, b):
    assert a.shape == b.shape and a.K == b.K
    assert _bits(a.ids) == _bits(b.ids) and _bits(a.probs) == _bits(b.probs)


def _pieces_equal(s, whole):
    from coda_b200.datasets import CompactSlab, ShardedCompactSlab
    pieces = [s] if isinstance(s, CompactSlab) else s.pieces
    offs = [0] if isinstance(s, CompactSlab) else s.offsets
    if not isinstance(s, CompactSlab):
        assert isinstance(s, ShardedCompactSlab)
    for p, off in zip(pieces, offs):
        assert p.device == DEV and p.ids.is_contiguous()
        _same_slab(p, whole.narrow_items(off, off + p.shape[1]))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shards", [1, 2, 3, 4])
def test_loader_equals_from_dense(tmp_path, dtype, shards):
    from coda_b200.datasets import load_compact
    from coda_b200.synth import shard_range
    H, N, C, K = 5, 1003, 37, 4
    x = _scores(H, N, C, seed=shards, dtype=dtype)
    p = str(tmp_path / "task.pt")
    torch.save(x.cpu(), p)
    whole = _from_dense(x, K)
    esz = x.element_size()
    for chunk in (1 << 20, C * esz, 7 * C * esz + 3, 50 * C * esz):   # one item per chunk, uneven splits
        s = load_compact(p, DEV, K, shards=shards, gpus=1, chunk_bytes=chunk)
        assert s.shape == (H, N, C)
        _pieces_equal(s, whole)
        if shards > 1:
            assert s.offsets == [shard_range(N, r, shards)[0] for r in range(shards)]
        assert torch.equal(s.compaction["flat_rows"].cpu(), whole.compaction["flat_rows"].cpu())
        assert _bits(s.compaction["dropped_max"]) == _bits(whole.compaction["dropped_max"])
    if dtype != torch.float32:                                    # a 16-bit file gives its fp32 widening's bits
        p32 = str(tmp_path / "task32.pt")
        torch.save(x.float().cpu(), p32)
        _same_slab(load_compact(p32, DEV, K), load_compact(p, DEV, K, chunk_bytes=3 * C * esz))


def test_saved_compact_file_reloads_to_the_same_bits(tmp_path):
    from coda import Dataset
    from coda_b200.datasets import ShardedCompactSlab, load_compact
    x = _scores(6, 777, 50, seed=3)
    whole = _from_dense(x, 3)
    p = str(tmp_path / "comp.pt")
    whole.save(p)
    for shards in (1, 2, 3):
        s = load_compact(p, DEV, shards=shards, gpus=1)
        assert s.compaction is None
        _pieces_equal(s, whole)
    with pytest.raises(ValueError, match="K = 3"):
        load_compact(p, DEV, 4)
    ds = Dataset(p, DEV)                                          # the shim: compact with no setting
    _pieces_equal(ds.preds, whole)
    s3 = load_compact(p, DEV, shards=3, gpus=1)
    assert isinstance(s3, ShardedCompactSlab)


def _requested(key):
    return torch.cuda.memory_stats(DEV)[f"requested_bytes.all.{key}"]


def test_load_holds_no_more_than_the_pieces_and_one_chunk(tmp_path):
    """Peak of the bytes the loader's tensors request, not of the allocator's blocks: a cached block reused without a
    split counts whole in ``max_memory_allocated`` (up to 1 MiB more than asked for), so that figure depends on what
    earlier work left in the cache, not on what the loader holds."""
    from coda_b200.datasets import load_compact
    H, N, C, K = 16, 20011, 100, 4
    p = str(tmp_path / "t.pt")
    torch.save(_scores(H, N, C, seed=9, dtype=torch.float16).cpu(), p)
    chunk = 3 << 16
    for cached in (False, True):                        # a fresh cache, then one with free holes from earlier work
        keep = []
        if cached:                                      # 2.3 MB holes between live blocks: a 1.7 MB piece reuses one unsplit
            holes = []
            for _ in range(3):
                holes.append(torch.empty(2300000, dtype=torch.uint8, device=DEV))
                keep.append(torch.empty(1100000, dtype=torch.uint8, device=DEV))
            del holes
        torch.cuda.synchronize()
        base = _requested("current")
        torch.cuda.reset_peak_memory_stats(DEV)
        s = load_compact(p, DEV, K, shards=3, gpus=1, chunk_bytes=chunk)
        peak = _requested("peak") - base
        held = sum(q.ids.numel() * 6 for q in s.pieces)
        small = 4 * H * (4 + 8) + 64                    # per-model diagnostics, their merge and the flags word
        assert held <= peak <= held + chunk + small, (peak, held, cached)
        del s, keep


# ------------------------------------------------------------------------------------------------------------------
# true losses
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N", [1, 7, 1000, 65537, 333331])
def test_true_losses_have_the_dense_bits(N):
    from coda.options import LOSS_FNS
    from coda_b200 import Oracle, TensorDataset
    from coda_b200.datasets import ShardedCompactSlab
    from coda_b200.synth import shard_range
    H, C = (7, 10) if N < 100000 else (3, 5)
    x = _scores(H, N, C, seed=N)
    labels = torch.randint(0, C, (N,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(N))
    want = Oracle(TensorDataset(x, labels), loss_fn=LOSS_FNS["acc"]).true_losses(x)
    whole = _from_dense(x, 4)
    got = Oracle(TensorDataset(whole, labels), loss_fn=LOSS_FNS["acc"]).true_losses(whole)
    assert got.dtype == torch.float32 and _bits(got) == _bits(want)
    for k in (2, 3):
        k = min(k, N)
        if k < 2:
            continue
        s = ShardedCompactSlab([whole.narrow_items(*shard_range(N, r, k)).to(DEV) for r in range(k)])
        got = Oracle(TensorDataset(s, labels), loss_fn=LOSS_FNS["acc"]).true_losses(s)
        assert _bits(got) == _bits(want), (N, k)


def test_a_flat_row_is_counted_where_densify_moves_the_arg_max():
    from coda.options import LOSS_FNS
    from coda_b200 import Oracle, TensorDataset
    x = torch.full((1, 3, 10), 0.89 / 9, device=DEV)
    x[0, 0, 7] = 0.11                                             # K = 1: rest = 0.89 / 9 < 0.11
    x[0, 1] = 0.05                                                # near-uniform: rest = 0.94 / 9 > 0.06
    x[0, 1, 5] = 0.06
    x[0, 2] = 0.0
    x[0, 2, 3] = 1.0
    s = _from_dense(x, 1)
    assert s.ids[0, :, 0].tolist() == [7, 5, 3]
    assert s.compaction["flat_rows"].tolist() == [1]
    d = s.densify()
    assert d[0].argmax(-1).tolist() == [7, 0, 3]                  # the flat row's arg-max is a remainder class
    labels = torch.tensor([7, 5, 3], device=DEV)
    orc = lambda p: Oracle(TensorDataset(p, labels), loss_fn=LOSS_FNS["acc"]).true_losses(p)
    assert _bits(orc(s)) == _bits(orc(x)) and float(orc(s)[0]) == 0.0
    assert float(orc(d)[0]) > 0.0                                 # densify() differs there, and only there


# ------------------------------------------------------------------------------------------------------------------
# pieces equal one slab
# ------------------------------------------------------------------------------------------------------------------
def _compact_task(H=24, N=1500, C=30, K=4, seed=11):
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, seed)
    return _from_dense(preds.to(DEV), K), labels


def _sharded(whole, k):
    from coda_b200.datasets import ShardedCompactSlab
    from coda_b200.synth import shard_range
    N = whole.shape[1]
    return ShardedCompactSlab([whole.narrow_items(*shard_range(N, r, k)).to(DEV) for r in range(k)])


def _same_state(a, b):
    assert torch.equal(a.dirichlets, b.dirichlets) and torch.equal(a.pi_hat, b.pi_hat)
    assert torch.equal(a.get_pbest(), b.get_pbest()) and torch.equal(a.pi_hat_xi, b.pi_hat_xi)


@pytest.mark.parametrize("k", [2, 3])
def test_coda_api_on_compact_pieces_equals_shards_on_one_slab(k):
    from coda_b200 import CODA, TensorDataset
    whole, labels = _compact_task()
    lab = labels.to(DEV)
    random.seed(0)
    ref = CODA(TensorDataset(whole, lab), shards=k)
    s = _sharded(whole, k)
    pcs = CODA(TensorDataset(s, lab))
    assert len(pcs.engines) == k and [e.preds.ids.data_ptr() for e in pcs.engines] == [p.ids.data_ptr() for p in s.pieces]
    _same_state(ref, pcs)
    for _ in range(8):
        st = random.getstate()
        i1, q1 = ref.get_next_item_to_label()
        after = random.getstate()
        random.setstate(st)
        i2, q2 = pcs.get_next_item_to_label()
        assert (i1, q1) == (i2, q2) and random.getstate() == after
        ref.add_label(i1, int(labels[i1]), q1)
        pcs.add_label(i2, int(labels[i2]), q2)
        assert int(ref.get_best_model_prediction()) == int(pcs.get_best_model_prediction())
        _same_state(ref, pcs)
    one = CODA(TensorDataset(whole, lab))
    one.load_state_dict(pcs.state_dict())                          # pieces -> one slab
    _same_state(pcs, one)


@pytest.mark.parametrize("kw", [{}, {"q": "iid"}, {"q": "uncertainty"}, {"prefilter_n": 50}])
@pytest.mark.parametrize("tie_rule", ["first", "reference"])
def test_coda_run_steps_on_compact_pieces(kw, tie_rule):
    from coda_b200 import CODA, TensorDataset
    whole, labels = _compact_task()
    lab = labels.to(DEV)
    for k in (2, 3):
        runs = []
        for ds, skw in ((TensorDataset(whole, lab), {"shards": k}), (TensorDataset(_sharded(whole, k), lab), {})):
            random.seed(5)
            sel = CODA(ds, **kw, **skw)
            sel.run_steps(10, lab, record_best=True, tie_rule=tie_rule)
            runs.append(([np.asarray(a).tobytes() for a in sel.history()], sel.best_history()[0].tolist(),
                         random.getstate(), sel.get_pbest().cpu().numpy().tobytes(), sel.pi_hat.cpu().numpy().tobytes()))
        assert runs[0] == runs[1], (kw, tie_rule, k)


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


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("method", ["iid", "uncertainty", "activetesting", "vma", "model_picker"])
def test_baselines_on_compact_pieces_equal_shards_on_one_slab(method, k):
    from coda_b200 import TensorDataset
    whole, labels = _compact_task(H=12, N=500, C=6, K=3, seed=3)
    lab = labels.to(DEV)
    for path, rule in (("api", None), ("loop", "philox"), ("loop", "reference")):
        runs = []
        for ds, kw in ((TensorDataset(whole, lab), {"shards": k}), (TensorDataset(_sharded(whole, k), lab), {})):
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
                sel.run_steps(15, lab, tie_rule=rule)
                tr = [np.asarray(a).tolist() for a in list(sel.history()) + list(sel.best_history())]
            post = getattr(sel, "posterior", None)
            runs.append((tr, torch.get_rng_state().numpy().tobytes(), torch.cuda.get_rng_state().numpy().tobytes(),
                         random.getstate(), None if post is None else post.cpu().numpy().tobytes()))
            sel.close()
        assert runs[0] == runs[1], (method, k, path, rule)


# ------------------------------------------------------------------------------------------------------------------
# near-lossless: K = C - 1 keeps every class
# ------------------------------------------------------------------------------------------------------------------
def test_k_equal_c_minus_one_follows_the_dense_run():
    from coda_b200 import CODA, TensorDataset
    g = load_golden("traj_tiny_h8_n300_c5")
    preds, labels = golden_slab(g)
    dense = preds.to(DEV)
    lab = labels.to(DEV)
    comp = _from_dense(dense, 4)
    random.seed(0)
    a = CODA(TensorDataset(dense, lab), **g["ctor"])
    random.seed(0)
    b = CODA(TensorDataset(comp, lab), **g["ctor"])
    assert torch.equal(a.engine.hard, b.engine.hard) and torch.equal(a.engine.disagree, b.engine.disagree)
    for step in range(int(g["steps"])):
        st = random.getstate()
        i, q = a.get_next_item_to_label()
        random.setstate(st)
        b.get_next_item_to_label()
        np.testing.assert_allclose(b.engine.eig.cpu().numpy(), a.engine.eig.cpu().numpy(), atol=5e-6)
        a.add_label(i, int(labels[i]), q)                        # teacher-forced: the dense run's pick for both
        b.add_label(i, int(labels[i]), q)
        np.testing.assert_allclose(b.pi_hat_xi.cpu().numpy(), a.pi_hat_xi.cpu().numpy(), rtol=1e-5, atol=1e-9)
        np.testing.assert_allclose(b.get_pbest().cpu().numpy(), a.get_pbest().cpu().numpy(), atol=1e-5)


# ------------------------------------------------------------------------------------------------------------------
# drop-in: main.py's calls through the shim with CODA_B200_COMPACT_K
# ------------------------------------------------------------------------------------------------------------------
_DRIVER = """\
import json
import random
import sys

import numpy as np
import torch

from coda import CODA, Dataset, Oracle
from coda.baselines import IID
from coda.options import LOSS_FNS

path, method, iters, out = sys.argv[1], sys.argv[2], int(sys.argv[3]), sys.argv[4]
random.seed(0); np.random.seed(0); torch.manual_seed(0); torch.cuda.manual_seed_all(0)
dataset = Dataset(path, device=torch.device("cuda"))
oracle = Oracle(dataset, loss_fn=LOSS_FNS["acc"])
true_losses = oracle.true_losses(dataset.preds)
best_loss = min(oracle.true_losses(dataset.preds))
if method == "coda":
    sel = CODA(dataset, prefilter_n=0, alpha=0.9, learning_rate=0.01, multiplier=2.0, disable_diag_prior=False, q="eig")
else:
    sel = IID(dataset, LOSS_FNS["acc"])
regrets = [float(true_losses[sel.get_best_model_prediction()] - best_loss)]
for step in range(iters):
    i, q = sel.get_next_item_to_label()
    sel.add_label(i, oracle(i), q)
    regrets.append(float(true_losses[sel.get_best_model_prediction()] - best_loss))
json.dump({"kind": type(dataset.preds).__name__, "regrets": regrets, "labeled": list(map(int, sel.labeled_idxs))
           if hasattr(sel, "labeled_idxs") else []}, open(out, "w"))
"""


def test_main_py_calls_through_the_shim_with_compaction(tmp_path):
    from coda.options import LOSS_FNS
    from coda_b200 import CODA, IID, Oracle, TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(16, 800, 12, 4)
    p = str(tmp_path / "task.pt")
    torch.save(preds, p)
    torch.save(labels, p.replace(".pt", "_labels.pt"))
    driver = str(tmp_path / "driver.py")
    with open(driver, "w") as f:
        f.write(_DRIVER)
    env = dict(os.environ, CODA_B200_COMPACT_K="4", PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "stubs")]),
               PYTHONSAFEPATH="1")
    whole = _from_dense(preds.to(DEV), 4)
    lab = labels.to(DEV)
    iters = 12
    for method in ("coda", "iid"):
        out = str(tmp_path / f"{method}.json")
        r = subprocess.run([sys.executable, driver, p, method, str(iters), out], env=env, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        got = json.load(open(out))
        assert got["kind"] == "CompactSlab"
        # the same calls in this process on CompactSlab.from_dense
        _seed(0)
        ds = TensorDataset(whole, lab)
        oracle = Oracle(ds, loss_fn=LOSS_FNS["acc"])
        tl = oracle.true_losses(whole)
        best = min(oracle.true_losses(whole))
        sel = CODA(ds) if method == "coda" else IID(ds, LOSS_FNS["acc"])
        regrets = [float(tl[sel.get_best_model_prediction()] - best)]
        for _ in range(iters):
            i, q = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), q)
            regrets.append(float(tl[sel.get_best_model_prediction()] - best))
        assert got["regrets"] == regrets, method
