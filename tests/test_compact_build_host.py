"""CPU checks of building and loading compact top-K slabs: the host model of the compaction kernel on crafted rows, the
row-aligned chunk walk, the compact file format through its memory map, ``ShardedCompactSlab``'s surface and refusals,
the shim's choice of load, and the ABI entries."""
import os
import re

import numpy as np
import pytest
import torch

from helpers import ROOT


def compact_host(x, K):
    """Host model of ``coda_b200_compact_build`` on an (H, N, C) float32 array (16-bit slabs: their fp32 widening).
    -> ids (H, N, K) int64, probs (H, N, K) float32, dropped_max (H,) float32, flat_rows (H,) int64.

    Per row the order is ``np.lexsort((class, -score))``: descending score, equal scores (-0.0 == 0.0) by ascending
    class.  ``dropped_max`` is the max of the (K+1)-th scores taken on their int32 bits, starting at +0.0 (the kernel's
    atomicMax on the bits: the float max for scores >= 0).  ``flat_rows`` counts rows whose remainder
    ``(1 - sum probs) * fp32(1 / (C - K))`` -- a left-to-right fp32 sum, as compact_rest forms it -- is >= probs[0]."""
    x = np.asarray(x, dtype=np.float32)
    H, N, C = x.shape
    ids = np.empty((H, N, K), dtype=np.int64)
    probs = np.empty((H, N, K), dtype=np.float32)
    dropped = np.zeros(H, dtype=np.int32)
    flat = np.zeros(H, dtype=np.int64)
    inv = np.float32(1.0) / np.float32(C - K)
    cls = np.arange(C)
    for h in range(H):
        for n in range(N):
            row = x[h, n]
            order = np.lexsort((cls, -row))
            ids[h, n] = order[:K]
            probs[h, n] = row[order[:K]]
            dropped[h] = max(dropped[h], row[order[K]:order[K] + 1].view(np.int32)[0])
            s = probs[h, n, 0]
            for j in range(1, K):
                s = np.float32(s + probs[h, n, j])
            rest = np.float32(np.float32(1.0) - s) * inv
            flat[h] += bool(rest >= probs[h, n, 0])
    return ids, probs, dropped.view(np.float32), flat


def _crafted_rows(C, K, rng):
    """Rows with all-equal scores, ties at the K-th place, -0.0 against 0.0, and plain random scores."""
    rows = [np.full(C, np.float32(1.0 / C)), np.zeros(C, np.float32), np.full(C, -0.0, np.float32)]
    t = rng.random(C).astype(np.float32) * np.float32(0.5)
    order = np.argsort(-t, kind="stable")
    t[order[K - 1:min(C, K + 2)]] = np.float32(0.25)          # a tie across the K-th place
    rows.append(t)
    z = np.where(rng.random(C) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
    z[rng.integers(C)] = np.float32(0.5)
    rows.append(z)
    rows.append(rng.random(C).astype(np.float32))
    q = (np.floor(rng.random(C) * 4) / 4).astype(np.float32)    # many exact ties
    rows.append(q)
    return np.stack(rows)[None]


@pytest.mark.parametrize("C,K", [(2, 1), (3, 2), (4, 3), (5, 4), (9, 8), (5, 1), (10, 4), (33, 8), (100, 3)])
def test_host_model_on_crafted_rows(C, K):
    rng = np.random.default_rng(C * 10 + K)
    x = _crafted_rows(C, K, rng)
    ids, probs, dropped, flat = compact_host(x, K)
    for n in range(x.shape[1]):
        row = x[0, n]
        want = sorted(range(C), key=lambda c: (-float(row[c]), c))          # -0.0 == 0.0: the class decides
        assert ids[0, n].tolist() == want[:K]
        assert probs[0, n].view(np.int32).tolist() == row[want[:K]].view(np.int32).tolist()   # the bits, -0.0 kept
        assert ids[0, n, 0] == int(np.argmax(row))                            # torch.argmax's first maximum
    assert ids[0, 0].tolist() == list(range(K))                               # all equal: the lowest classes
    assert ids[0, 2].tolist() == list(range(K)) and np.signbit(probs[0, 2]).all()
    drops = [x[0, n][sorted(range(C), key=lambda c: (-float(x[0, n][c]), c))[K]] for n in range(x.shape[1])]
    assert dropped[0] == max(max(drops), 0.0) and not np.signbit(dropped[0])
    assert 2 <= flat[0] <= x.shape[1]                                         # the all-zero rows: rest 1/(C-K) > 0
    one = np.zeros((1, 1, C), np.float32)
    one[0, 0, C - 1] = 1.0
    assert compact_host(one, K)[3][0] == 0                                    # a confident row is not flat


def test_host_model_keeps_every_class_at_k_equal_c_minus_one():
    rng = np.random.default_rng(1)
    x = rng.random((2, 40, 5)).astype(np.float32)
    ids, probs, _, _ = compact_host(x, 4)
    for h in range(2):
        for n in range(40):
            missing = ({0, 1, 2, 3, 4} - set(ids[h, n].tolist())).pop()
            assert x[h, n, missing] <= probs[h, n].min()


@pytest.mark.parametrize("lo,hi,C,esz,chunk", [(0, 10, 3, 4, 8), (0, 10, 3, 4, 12), (5, 9, 100, 2, 64), (0, 1, 1, 4, 1),
                                               (3, 40, 7, 4, 1 << 20), (2, 3, 4096, 4, 1000), (7, 1000, 10, 2, 333)])
def test_row_walk_takes_whole_items_and_covers_the_range(lo, hi, C, esz, chunk):
    from coda_b200.datasets import row_walk
    w = row_walk(lo, hi, C, esz, chunk)
    assert w[0][0] == lo and w[-1][1] == hi
    assert all(a[1] == b[0] for a, b in zip(w, w[1:]))
    assert all(b - a >= 1 for a, b in w)                                      # at least one item per chunk
    per = max(1, chunk // (C * esz))
    assert all(b - a <= per for a, b in w) and all(b - a == per for a, b in w[:-1])
    assert all((b - a) * C * esz <= chunk for a, b in w) or per == 1


def _compact_cpu(H=3, N=11, C=9, K=4, seed=0):
    from coda_b200.datasets import CompactSlab
    g = torch.Generator().manual_seed(seed)
    ids = torch.stack([torch.randperm(C, generator=g)[:K] for _ in range(H * N)]).view(H, N, K).to(torch.int16)
    probs = torch.rand(H, N, K, generator=g).sort(-1, descending=True).values / K
    return CompactSlab(ids, probs, C)


def test_compact_file_round_trip_through_the_memory_map(tmp_path):
    from coda_b200.datasets import _open_compact, is_compact_file
    s = _compact_cpu()
    p = str(tmp_path / "c.pt")
    s.save(p)
    assert is_compact_file(p)
    obj = _open_compact(p)
    assert obj["format"] == "coda_b200.compact" and obj["version"] == 1 and obj["C"] == 9
    assert torch.equal(obj["ids"], s.ids) and obj["probs"].numpy().tobytes() == s.probs.numpy().tobytes()
    assert obj["ids"][1, 3:7].numpy().tobytes() == s.ids[1, 3:7].numpy().tobytes()     # a piece's range of one model
    # a view saves as its own contiguous slab
    v = s.narrow_items(2, 8)
    v.save(p)
    assert torch.equal(_open_compact(p)["ids"], s.ids[:, 2:8]) and _open_compact(p)["ids"].is_contiguous()
    d = str(tmp_path / "d.pt")
    torch.save(torch.rand(2, 3, 4), d)
    assert not is_compact_file(d) and _open_compact(d) is None
    torch.save(torch.rand(2, 3, 4), d, _use_new_zipfile_serialization=False)
    assert not is_compact_file(d)
    torch.save({"format": "coda_b200.compact", "version": 2, "ids": s.ids, "probs": s.probs, "C": 9}, d)
    with pytest.raises(ValueError, match="version"):
        _open_compact(d)


def test_compact_k_is_checked():
    from coda_b200.datasets import _check_k
    for K, C in [(4, 4), (5, 100), (0, 10), (None, 10), (16, 100), (4, 4097)]:
        with pytest.raises(ValueError):
            _check_k(K, C)
    assert [_check_k(k, 9) for k in (1, 2, 3, 4, 8)] == [1, 2, 3, 4, 8]


def test_sharded_compact_slab_attributes_and_refusals():
    from coda_b200.datasets import CompactSlab, ShardedCompactSlab, ShardedSlab
    whole = _compact_cpu(H=2, N=12, C=7, K=3)
    ps = [whole.narrow_items(0, 4), whole.narrow_items(4, 7), whole.narrow_items(7, 12)]
    s = ShardedCompactSlab(ps)
    assert s.shape == (2, 12, 7) and s.offsets == [0, 4, 7] and s.K == 3 and s.C == 7
    assert s.dtype == torch.float32 and not s.is_cuda and s.device == ps[0].device and s.numel() == whole.numel()
    assert [off for _, off in s.layout()] == [0, 4, 7] and [p for p, _ in s.layout()] == ps
    for i in range(12):
        assert s.item_column(i).numpy().tobytes() == whole.item_column(i).numpy().tobytes()
    with pytest.raises(IndexError):
        s.item_column(12)
    with pytest.raises(TypeError, match="compact"):
        ShardedSlab([whole])                                      # the dense class keeps refusing compact pieces
    with pytest.raises(TypeError, match="dense"):
        ShardedCompactSlab([torch.rand(2, 3, 7)])
    with pytest.raises(TypeError):
        ShardedCompactSlab([ps[0], _compact_cpu(H=2, N=4, C=7, K=4)])     # mixed K
    with pytest.raises(TypeError):
        ShardedCompactSlab([ps[0], _compact_cpu(H=3, N=4, C=7, K=3)])     # mixed H
    with pytest.raises(TypeError):
        ShardedCompactSlab([ps[0], _compact_cpu(H=2, N=4, C=8, K=3)])     # mixed C
    with pytest.raises(ValueError):
        ShardedCompactSlab([ps[0], whole.narrow_items(5, 5)])             # an empty piece
    with pytest.raises(ValueError):
        ShardedCompactSlab([])
    assert isinstance(ps[0], CompactSlab)


class _World2:
    world, rank = 2, 0


def test_selectors_refuse_a_layout_that_disagrees_with_the_compact_pieces():
    from coda_b200 import CODA, IID, ModelPicker, TensorDataset
    from coda_b200.datasets import ShardedCompactSlab
    whole = _compact_cpu(H=2, N=12, C=7, K=3)
    s = ShardedCompactSlab([whole.narrow_items(0, 4), whole.narrow_items(4, 7), whole.narrow_items(7, 12)])
    ds = TensorDataset(s, torch.zeros(12, dtype=torch.int64))
    makers = (lambda **kw: CODA(ds, **kw), lambda **kw: IID(ds, None, **kw), lambda **kw: ModelPicker(ds, **kw))
    for make in makers:
        for kw in ({"shards": 2}, {"gpus": 2}, {"shards": 4}, {"shards": 3, "gpus": 2}):
            with pytest.raises(ValueError, match="disagrees"):
                make(**kw)
        with pytest.raises(ValueError, match="torch.distributed"):
            make(comm=_World2())


def test_eps_search_and_true_losses_refuse_what_they_do_not_take():
    from coda.options import LOSS_FNS
    from coda_b200 import Oracle, TensorDataset
    from coda_b200.datasets import ShardedCompactSlab
    from coda_b200.eps_search import modelpicker_eps_search
    whole = _compact_cpu(H=2, N=12, C=7, K=3)
    s = ShardedCompactSlab([whole.narrow_items(0, 5), whole.narrow_items(5, 12)])
    with pytest.raises(NotImplementedError, match="ShardedCompactSlab"):
        modelpicker_eps_search(TensorDataset(s, None))
    labels = torch.zeros(12, dtype=torch.int64)
    for slab in (s, whole):
        with pytest.raises(NotImplementedError, match="accuracy loss"):
            Oracle(TensorDataset(slab, labels), loss_fn=torch.nn.functional.cross_entropy).true_losses(slab)
        with pytest.raises(NotImplementedError, match="1-D"):
            Oracle(TensorDataset(slab, torch.zeros(12, 7)), loss_fn=LOSS_FNS["acc"]).true_losses(slab)
        with pytest.raises(NotImplementedError, match="CUDA"):
            Oracle(TensorDataset(slab, labels), loss_fn=LOSS_FNS["acc"]).true_losses(slab)


# ---------------------------------------------------------------------------------------------------------------------
# the shim's choice of load
# ---------------------------------------------------------------------------------------------------------------------
def _count(monkeypatch, path, env, free, ngpus, K=None, device="cuda:0"):
    """``load_route``'s piece count of a compact load (0 for one piece)."""
    import coda_b200.datasets as ds
    monkeypatch.setattr(ds, "_free_bytes", lambda index: free)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: ngpus)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    route = ds.load_route(path, device, {**env, **({"CODA_B200_COMPACT_K": str(K)} if K else {})})
    assert route["compact_k"] == K
    return route["shards"] or 0


def test_load_route_compact_piece_count(tmp_path, monkeypatch):
    dense = str(tmp_path / "task.pt")
    torch.save(torch.rand(4, 50, 10), dense)
    comp = str(tmp_path / "comp.pt")
    _compact_cpu(H=4, N=50, C=10, K=3).save(comp)
    b4 = 4 * 50 * 4 * 6                                           # the dense file compacted at K = 4
    b3 = 4 * 50 * 3 * 6                                           # the saved K = 3 slab
    assert _count(monkeypatch, dense, {"CODA_B200_SHARD_LOAD": "1"}, 1 << 40, 1, K=4) == 1
    assert _count(monkeypatch, dense, {"CODA_B200_SHARD_LOAD": "1"}, 1 << 40, 4, K=4) == 4
    assert _count(monkeypatch, comp, {"CODA_B200_SHARD_LOAD": "1", "CODA_B200_GPUS": "3"}, 1 << 40, 1) == 3
    assert _count(monkeypatch, dense, {}, b4 - 1, 2, K=4) == 2
    assert _count(monkeypatch, dense, {}, b4, 2, K=4) == 0
    assert _count(monkeypatch, dense, {}, b4 - 1, 1, K=4) == 0
    assert _count(monkeypatch, comp, {}, b3 - 1, 2) == 2
    assert _count(monkeypatch, comp, {}, b3, 2) == 0
    assert _count(monkeypatch, comp, {"CODA_B200_GPUS": "8"}, 0, 4) == 8
    assert _count(monkeypatch, comp, {}, 0, 4, device="cpu") == 0


def _shim_calls(monkeypatch, path, env):
    import coda_b200.datasets as ds
    from coda.datasets import Dataset
    for k in ("CODA_B200_COMPACT_K", "CODA_B200_SHARD_LOAD", "CODA_B200_GPUS", "CODA_B200_KEEP_DTYPE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: 1)
    calls = []
    monkeypatch.setattr(ds.Dataset, "__init__", lambda self, *a, **kw: calls.append((a, kw)))
    Dataset(path, "cuda:0")
    return calls


def test_shim_choice_of_load(tmp_path, monkeypatch):
    dense = str(tmp_path / "task.pt")
    torch.save(torch.rand(4, 50, 10), dense)
    comp = str(tmp_path / "comp.pt")
    _compact_cpu(H=4, N=50, C=10, K=3).save(comp)
    # a dense file without the variable: exactly the call it got before
    assert _shim_calls(monkeypatch, dense, {}) == [((dense, "cuda:0"), {"keep_dtype": False})]
    assert _shim_calls(monkeypatch, dense, {"CODA_B200_KEEP_DTYPE": "1"}) == [((dense, "cuda:0"), {"keep_dtype": True})]
    assert _shim_calls(monkeypatch, dense, {"CODA_B200_SHARD_LOAD": "1", "CODA_B200_GPUS": "2"}) == \
        [((dense, "cuda:0"), {"keep_dtype": False, "shards": 2})]
    # opt-in compaction of a dense file, one piece or CODA_B200_GPUS pieces
    assert _shim_calls(monkeypatch, dense, {"CODA_B200_COMPACT_K": "4"}) == \
        [((dense, "cuda:0"), {"compact_k": 4, "shards": None})]
    assert _shim_calls(monkeypatch, dense, {"CODA_B200_COMPACT_K": "4", "CODA_B200_SHARD_LOAD": "1",
                                            "CODA_B200_GPUS": "3"}) == [((dense, "cuda:0"), {"compact_k": 4, "shards": 3})]
    # a saved compact slab loads as compact with no setting
    assert _shim_calls(monkeypatch, comp, {}) == [((comp, "cuda:0"), {"compact_k": None, "shards": None})]
    assert _shim_calls(monkeypatch, comp, {"CODA_B200_SHARD_LOAD": "1"}) == \
        [((comp, "cuda:0"), {"compact_k": None, "shards": 1})]


# ---------------------------------------------------------------------------------------------------------------------
# ABI
# ---------------------------------------------------------------------------------------------------------------------
def test_compact_build_abi_entries_are_declared_exported_and_bound():
    from coda_b200 import _native as nat
    from coda_b200 import build
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    for name, n in (("coda_b200_compact_build", 14), ("coda_b200_true_loss_counts_compact", 8)):
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
        assert m and m.group(1).count(",") + 1 == n == len(nat.SIGNATURES[name][1]), name
        assert hasattr(nat.load(), name)
    assert nat.load().coda_b200_version() == 203 == nat.VERSION
    assert "compact_build.cu" in build.SOURCES
    pre = open(os.path.join(ROOT, "coda_b200", "csrc", "preload.cu")).read()
    assert "coda_anchor_compact_build()" in pre
