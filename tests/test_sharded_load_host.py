"""CPU checks of loading a slab as N-range pieces (``ShardedSlab``): the piece plan, the shim's decision rule, the
refusals that need no device, and the ABI entry of the true-loss pass."""
import os
import re

import pytest
import torch

from helpers import ROOT


def _slab_file(tmp_path, H=3, N=11, C=4, dtype=torch.float32, legacy=False):
    p = str(tmp_path / "task.pt")
    t = torch.rand(H, N, C).to(dtype)
    if legacy:
        torch.save(t, p, _use_new_zipfile_serialization=False)
    else:
        torch.save(t, p)
    return p, t


@pytest.mark.parametrize("N,nshards,ngpus,ndev,home", [(10, 1, 1, 1, 0), (11, 3, 1, 1, 0), (1000, 4, 4, 8, 2),
                                                     (7, 5, 2, 2, 1), (100003, 8, 3, 4, 3), (5, 5, 5, 5, 0)])
def test_piece_plan_follows_split_slab(N, nshards, ngpus, ndev, home):
    from coda_b200.datasets import piece_plan
    from coda_b200.synth import shard_range
    plan = piece_plan(N, nshards, ngpus, home, ndev)
    assert [(lo, hi) for lo, hi, _ in plan] == [shard_range(N, r, nshards) for r in range(nshards)]
    assert plan[0][0] == 0 and plan[-1][1] == N and all(a[1] == b[0] for a, b in zip(plan, plan[1:]))
    devs = [d for _, _, d in plan]
    assert devs[0] == home
    # split_slab's rule: home first, then the others in order, consecutive pieces share a device
    order = [home] + [d for d in range(ndev) if d != home]
    order = order[:max(1, ngpus)]
    assert devs == [order[r * len(order) // nshards] for r in range(nshards)]
    assert devs == sorted(devs, key=order.index)


@pytest.mark.parametrize("lo,hi,C,esz,chunk", [(0, 10, 3, 4, 8), (5, 9, 100, 2, 64), (0, 1, 1, 4, 1), (3, 40, 7, 4, 1 << 20),
                                               (2, 3, 4096, 4, 1000)])
def test_chunk_walk_covers_one_models_range_contiguously(lo, hi, C, esz, chunk):
    from coda_b200.datasets import chunk_walk
    w = chunk_walk(lo, hi, C, esz, chunk)
    assert w[0][0] == lo * C and w[-1][1] == hi * C
    assert all(a[1] == b[0] for a, b in zip(w, w[1:]))
    assert all(0 < (b - a) * esz <= max(chunk, esz) for a, b in w)


def test_legacy_format_is_refused(tmp_path):
    from coda_b200.datasets import load_sharded
    p, _ = _slab_file(tmp_path, legacy=True)
    with pytest.raises(ValueError, match="legacy format"):
        load_sharded(p, "cuda:0", shards=2)


def test_non_contiguous_file_is_refused_with_a_message(tmp_path):
    from coda_b200.datasets import load_sharded
    p = str(tmp_path / "t.pt")
    torch.save(torch.rand(5, 3, 4).transpose(0, 1), p)
    with pytest.raises(ValueError, match="not contiguous"):
        load_sharded(p, "cuda:0", shards=2)


def _decide(monkeypatch, path, env, free, ngpus, keep=False, device="cuda:0"):
    """``load_route``'s device-piece count (0 for a plain load), with the host rules off (``CODA_B200_HOST_SLAB=0``)."""
    import coda_b200.datasets as ds
    monkeypatch.setattr(ds, "_free_bytes", lambda index: free)
    monkeypatch.setattr(torch.cuda, "device_count", lambda: ngpus)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    env = {"CODA_B200_HOST_SLAB": "0", "CODA_B200_KEEP_DTYPE": "1" if keep else "0", **env}
    route = ds.load_route(path, device, env)
    assert route["keep_dtype"] == keep and "host" not in route
    return route.get("shards", 0)


def test_load_route_device_piece_count(tmp_path, monkeypatch):
    p, t = _slab_file(tmp_path, H=4, N=50, C=10, dtype=torch.float16)
    b32 = t.numel() * 4
    b16 = t.numel() * 2
    # opt-in: CODA_B200_GPUS, else every visible GPU
    assert _decide(monkeypatch, p, {"CODA_B200_SHARD_LOAD": "1"}, 1 << 40, 1) == 1
    assert _decide(monkeypatch, p, {"CODA_B200_SHARD_LOAD": "1"}, 1 << 40, 4) == 4
    assert _decide(monkeypatch, p, {"CODA_B200_SHARD_LOAD": "1", "CODA_B200_GPUS": "3"}, 1 << 40, 1) == 3
    # automatic: only when the slab (held at fp32, or at its stored width when kept) exceeds the free memory AND > 1 GPU
    assert _decide(monkeypatch, p, {}, b32 - 1, 2) == 2
    assert _decide(monkeypatch, p, {}, b32, 2) == 0
    assert _decide(monkeypatch, p, {}, b32 - 1, 1) == 0
    assert _decide(monkeypatch, p, {}, b32 - 1, 2, keep=True) == 0
    assert _decide(monkeypatch, p, {}, b16 - 1, 2, keep=True) == 2
    assert _decide(monkeypatch, p, {"CODA_B200_GPUS": "8"}, 0, 4) == 8
    assert _decide(monkeypatch, p, {}, 0, 4, device="cpu") == 0
    assert _decide(monkeypatch, p, {"CODA_B200_SHARD_LOAD": "0"}, 1 << 40, 4) == 0


def test_load_route_device_pieces_keep_the_plain_load_for_a_legacy_file(tmp_path, monkeypatch):
    p, _ = _slab_file(tmp_path, legacy=True)
    assert _decide(monkeypatch, p, {}, 0, 4) == 0


def _pieces(dtype=torch.float32, ns=(4, 3, 5), H=2, C=3, device="cpu"):
    return [torch.rand(H, n, C, device=device).to(dtype) for n in ns]


def test_sharded_slab_attributes_and_refusals():
    from coda_b200.datasets import CompactSlab, ShardedSlab
    ps = _pieces(torch.float16)
    s = ShardedSlab(ps)
    assert s.shape == torch.Size([2, 12, 3]) and s.offsets == [0, 4, 7] and s.dtype == torch.float16
    assert s.numel() == 72 and s.element_size() == 2 and not s.is_cuda and s.device == ps[0].device
    full = torch.cat(ps, 1)
    for i in range(12):
        assert torch.equal(s.item_column(i), full[:, i].float())
    with pytest.raises(IndexError):
        s.item_column(12)
    compact = CompactSlab(torch.zeros(2, 4, 2, dtype=torch.int16), torch.zeros(2, 4, 2), 5)
    with pytest.raises(TypeError, match="compact"):
        ShardedSlab([compact])
    with pytest.raises(TypeError):
        ShardedSlab([ps[0], ps[1].float()])
    with pytest.raises(TypeError):
        ShardedSlab([torch.zeros(2, 3, 3, dtype=torch.float64)])
    with pytest.raises(TypeError):
        ShardedSlab([ps[0], torch.rand(2, 3, 4).half()])
    with pytest.raises(ValueError):
        ShardedSlab([torch.rand(2, 6, 3)[:, ::2]])
    with pytest.raises(ValueError):
        ShardedSlab([])


class _World2:
    world, rank = 2, 0


def test_selectors_refuse_a_layout_that_disagrees_with_the_pieces():
    from coda_b200 import CODA, IID, ModelPicker, TensorDataset
    from coda_b200.datasets import ShardedSlab
    s = ShardedSlab(_pieces())
    ds = TensorDataset(s, torch.zeros(12, dtype=torch.int64))
    makers = (lambda **kw: CODA(ds, **kw), lambda **kw: IID(ds, None, **kw), lambda **kw: ModelPicker(ds, **kw))
    for make in makers:
        for kw in ({"shards": 2}, {"gpus": 2}, {"shards": 4}, {"shards": 3, "gpus": 2}):
            with pytest.raises(ValueError, match="disagrees"):
                make(**kw)
        with pytest.raises(ValueError, match="torch.distributed"):
            make(comm=_World2())


def test_eps_search_refuses_a_sharded_slab():
    from coda_b200 import TensorDataset
    from coda_b200.datasets import ShardedSlab
    from coda_b200.eps_search import modelpicker_eps_search
    with pytest.raises(NotImplementedError, match="ShardedSlab"):
        modelpicker_eps_search(TensorDataset(ShardedSlab(_pieces()), None))


def test_true_losses_on_pieces_refuse_what_they_do_not_compute():
    from coda.options import LOSS_FNS
    from coda_b200 import Oracle, TensorDataset
    from coda_b200.datasets import ShardedSlab
    s = ShardedSlab(_pieces())
    labels = torch.zeros(12, dtype=torch.int64)
    with pytest.raises(NotImplementedError, match="accuracy loss"):
        Oracle(TensorDataset(s, labels), loss_fn=torch.nn.functional.cross_entropy).true_losses(s)
    with pytest.raises(NotImplementedError, match="1-D"):
        Oracle(TensorDataset(s, torch.zeros(12, 3)), loss_fn=LOSS_FNS["acc"]).true_losses(s)
    big = ShardedSlab([torch.empty(1, 1 << 23, 1, device="meta"), torch.empty(1, 1 << 23, 1, device="meta")])
    with pytest.raises(NotImplementedError, match="2\\^24"):
        Oracle(TensorDataset(big, labels), loss_fn=LOSS_FNS["acc"]).true_losses(big)
    ok = ShardedSlab([torch.empty(1, (1 << 24) - 1, 1, device="meta")])
    with pytest.raises(NotImplementedError, match="CUDA"):
        Oracle(TensorDataset(ok, labels), loss_fn=LOSS_FNS["acc"]).true_losses(ok)


def test_mean_factor_is_torchs():
    """float(H) / float(H*N) in fp32; on the CPU torch divides the sum instead, so this only pins the arithmetic (the
    GPU tier checks the bits against torch's CUDA mean)."""
    import numpy as np
    from coda_b200.oracle import mean_factor
    for H, N in [(1, 3), (80, 10000), (256, 1000000), (7, 16777215), (1024, 999983)]:
        f = mean_factor(H, N)
        assert f.dtype == np.float32 and f == np.float32(np.float32(H) / np.float32(float(H * N)))


def test_true_loss_abi_entry_is_declared_and_exported():
    from coda_b200 import _native as nat
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    for name, n in (("coda_b200_true_loss_counts", 9), ("coda_b200_preload_kernels", 1)):
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
        assert m and m.group(1).count(",") + 1 == n == len(nat.SIGNATURES[name][1]), name
        assert hasattr(nat.load(), name)
    assert nat.load().coda_b200_version() == 203
    from coda_b200 import build
    assert "true_loss.cu" in build.SOURCES and "preload.cu" in build.SOURCES


def test_every_translation_unit_with_kernels_names_an_anchor():
    """coda_b200_preload_kernels reaches a unit's kernels through its CODA_MODULE_ANCHOR: a unit with kernels and no
    anchor would be left to lazy loading."""
    from coda_b200 import build
    csrc = os.path.join(ROOT, "coda_b200", "csrc")
    pre = open(os.path.join(csrc, "preload.cu")).read()
    for f in build.SOURCES:
        src = open(os.path.join(csrc, f)).read()
        kernels = "__global__" in src or (f == "step_defer.cu")               # step_defer's kernel is in a header
        m = re.search(r"^CODA_MODULE_ANCHOR\((\w+), ", src, flags=re.M)
        assert bool(m) == kernels, f
        if m:
            assert m.group(1) == f[:-3] and f"coda_anchor_{m.group(1)}()" in pre, f
