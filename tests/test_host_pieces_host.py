"""CPU tier of a host-resident slab in N-range pieces (``ShardedHostSlab``): the load route's host-piece rule and its
dispatch, the N-range ``HostSlab`` view, the pieces' surface and validation, the loader's plan and its one shared memory
map, and the refusals that need no device."""
import pytest
import torch


def _slab_file(tmp_path, H=4, N=50, C=10, dtype=torch.float32):
    p = str(tmp_path / "task.pt")
    t = torch.rand(H, N, C).to(dtype)
    torch.save(t, p)
    return p, t


def _gpus(monkeypatch, free, current=0):
    """``free``: free bytes of each visible GPU, by index."""
    import coda_b200.datasets as ds
    monkeypatch.setattr(ds, "_free_bytes", lambda index: free[index])
    monkeypatch.setattr(torch.cuda, "device_count", lambda: len(free))
    monkeypatch.setattr(torch.cuda, "current_device", lambda: current)


def _count(monkeypatch, path, env, free, keep=False, device="cuda:0"):
    """How many host pieces ``load_route`` loads ``path`` into: 0 for none."""
    import coda_b200.datasets as ds
    _gpus(monkeypatch, free)
    route = ds.load_route(path, device, {"CODA_B200_KEEP_DTYPE": "1" if keep else "0", **env})
    return route["shards"] if route.get("host") and "shards" in route else 0


# ---------------------------------------------------------------------------------------------------------------------
# the shim's rule and its dispatch
# ---------------------------------------------------------------------------------------------------------------------
def test_load_route_host_piece_count(tmp_path, monkeypatch):
    p, t = _slab_file(tmp_path, dtype=torch.float16)
    b32, b16 = t.numel() * 4, t.numel() * 2
    # more than the summed free memory of the GPUs the pieces would use: one host piece per GPU
    assert _count(monkeypatch, p, {}, [b32 // 2, b32 // 2 - 1]) == 2
    assert _count(monkeypatch, p, {}, [b32 // 2, b32 // 2]) == 0            # fits across the two: device pieces
    assert _count(monkeypatch, p, {}, [b32 // 4] * 4) == 0
    assert _count(monkeypatch, p, {}, [b32 // 4 - 1] * 4) == 4
    assert _count(monkeypatch, p, {}, [0]) == 0                               # one GPU: HostSlab's rule instead
    assert _count(monkeypatch, p, {}, []) == 0
    assert _count(monkeypatch, p, {}, [0, 0], device="cpu") == 0
    # the width it would be held at
    assert _count(monkeypatch, p, {}, [b16, 0], keep=True) == 0
    assert _count(monkeypatch, p, {}, [b16 - 1, 0], keep=True) == 2
    assert _count(monkeypatch, p, {}, [b16 - 1, 0]) == 2
    # CODA_B200_GPUS pieces over the GPUs piece_plan picks: a GPU shared by several pieces counts once
    assert _count(monkeypatch, p, {"CODA_B200_GPUS": "3"}, [b32 // 2, b32 // 2 - 1]) == 3
    assert _count(monkeypatch, p, {"CODA_B200_GPUS": "3"}, [b32 // 2, b32 // 2]) == 0
    assert _count(monkeypatch, p, {"CODA_B200_GPUS": "1"}, [b32 - 1, 1 << 50]) == 1      # only the home GPU is used
    assert _count(monkeypatch, p, {"CODA_B200_GPUS": "2"}, [0, b32, 0, 0]) == 0          # GPUs 0 and 1
    assert _count(monkeypatch, p, {"CODA_B200_GPUS": "2"}, [0, 0, b32, b32]) == 2
    assert _count(monkeypatch, p, {"CODA_B200_GPUS": "2"}, [0, 0, b32, b32], device="cuda:2") == 0   # GPUs 2 and 0
    # either opt-in or opt-out keeps its own meaning; an empty value is unset
    for env in ({"CODA_B200_HOST_SLAB": "1"}, {"CODA_B200_HOST_SLAB": "0"}, {"CODA_B200_SHARD_LOAD": "1"},
                {"CODA_B200_SHARD_LOAD": "0"}):
        assert _count(monkeypatch, p, env, [0, 0]) == 0, env
    assert _count(monkeypatch, p, {"CODA_B200_HOST_SLAB": "", "CODA_B200_SHARD_LOAD": ""}, [0, 0]) == 2


def test_load_route_host_pieces_keep_the_plain_load_for_a_legacy_file(tmp_path, monkeypatch):
    p = str(tmp_path / "legacy.pt")
    torch.save(torch.rand(3, 11, 4), p, _use_new_zipfile_serialization=False)
    assert _count(monkeypatch, p, {}, [0, 0]) == 0


def _dispatch(tmp_path, monkeypatch, env, free, keep="0"):
    import coda_b200.datasets as ds
    from coda.datasets import Dataset
    p, _ = _slab_file(tmp_path)
    for k in ("CODA_B200_HOST_SLAB", "CODA_B200_SHARD_LOAD", "CODA_B200_GPUS", "CODA_B200_COMPACT_K"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("CODA_B200_KEEP_DTYPE", keep)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    _gpus(monkeypatch, free)
    calls = []
    monkeypatch.setattr(ds.Dataset, "__init__", lambda self, *a, **kw: calls.append((a, kw)))
    Dataset(p, "cuda:0")
    assert len(calls) == 1 and calls[0][0] == (p, "cuda:0")
    return calls[0][1]


def test_shim_dispatch(tmp_path, monkeypatch):
    b = 4 * 50 * 10 * 4
    d = lambda env, free, **kw: _dispatch(tmp_path, monkeypatch, env, free, **kw)   # noqa: E731
    # the new case: larger than every GPU together -> host pieces, one per GPU
    assert d({}, [b // 2, b // 2 - 1]) == {"keep_dtype": False, "host": True, "shards": 2}
    assert d({}, [0, 0, 0]) == {"keep_dtype": False, "host": True, "shards": 3}
    assert d({"CODA_B200_GPUS": "5"}, [0, 0]) == {"keep_dtype": False, "host": True, "shards": 5}
    assert d({}, [0, 0], keep="1") == {"keep_dtype": True, "host": True, "shards": 2}
    # every existing outcome
    assert d({}, [b // 2, b // 2]) == {"keep_dtype": False, "shards": 2}               # fits across the GPUs
    assert d({}, [1 << 50, 1 << 50]) == {"keep_dtype": False}                         # fits on one
    assert d({}, [0]) == {"keep_dtype": False, "host": True}                          # one GPU: one HostSlab
    assert d({}, [1 << 50]) == {"keep_dtype": False}
    assert d({"CODA_B200_HOST_SLAB": "1"}, [0, 0]) == {"keep_dtype": False, "host": True}
    assert d({"CODA_B200_HOST_SLAB": "0"}, [0, 0]) == {"keep_dtype": False, "shards": 2}
    assert d({"CODA_B200_HOST_SLAB": "0"}, [0]) == {"keep_dtype": False}
    assert d({"CODA_B200_SHARD_LOAD": "1"}, [0, 0]) == {"keep_dtype": False, "shards": 2}
    assert d({"CODA_B200_SHARD_LOAD": "1", "CODA_B200_GPUS": "3"}, [0, 0]) == {"keep_dtype": False, "shards": 3}
    kw = d({"CODA_B200_COMPACT_K": "2"}, [0, 0])                                       # compaction keeps precedence
    assert kw.get("compact_k") == 2 and "host" not in kw


# ---------------------------------------------------------------------------------------------------------------------
# the N-range HostSlab view and the pieces
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_host_slab_takes_an_n_range_view(dtype):
    from coda_b200 import HostSlab
    t = torch.rand(4, 1001, 6).to(dtype)
    for lo, hi in ((0, 1), (3, 700), (999, 1001), (0, 1001)):
        s = HostSlab(t[:, lo:hi], "cuda:0", chunk_items=100)
        assert s.shape == (4, hi - lo, 6) and s.host.data_ptr() == t.data_ptr() + lo * 6 * t.element_size()
        assert s.chunk_items == min(128, (hi - lo + 31) // 32 * 32)
    assert HostSlab(t[:1, 5:9], "cuda:0").shape == (1, 4, 6)
    for bad in (t.transpose(0, 1), t[:, ::2], t[:, :, :3], t[:, 5:5], t.transpose(1, 2)):
        with pytest.raises(ValueError):
            HostSlab(bad, "cuda:0")


def _host_pieces(dtype=torch.float32, ns=(4, 3, 5), H=2, C=3, devices=(0, 0, 1)):
    from coda_b200 import HostSlab
    full = torch.rand(H, sum(ns), C).to(dtype)
    pieces, lo = [], 0
    for n, d in zip(ns, devices):
        pieces.append(HostSlab(full[:, lo:lo + n], torch.device("cuda", d)))
        lo += n
    return full, pieces


def test_sharded_host_slab_surface_and_validation():
    from coda_b200 import HostSlab, ShardedHostSlab, ShardedSlab
    full, ps = _host_pieces(torch.float16)
    s = ShardedHostSlab(ps)
    assert s.shape == torch.Size([2, 12, 3]) and s.offsets == [0, 4, 7] and s.dtype == torch.float16
    assert s.numel() == 72 and s.element_size() == 2 and s.is_cuda and s.device == torch.device("cuda", 0)
    assert s.layout() == list(zip(ps, [0, 4, 7]))
    with pytest.raises(IndexError):
        s.item_column(12)
    with pytest.raises(IndexError):
        s.item_column(-1)
    widened = ShardedHostSlab([HostSlab(p.host, p.device, dtype=torch.float32) for p in ps])
    assert widened.dtype == torch.float32 and widened.element_size() == 4
    with pytest.raises(ValueError):
        ShardedHostSlab([])
    with pytest.raises(TypeError, match="HostSlab"):
        ShardedHostSlab([full])
    with pytest.raises(TypeError):
        ShardedHostSlab([ps[0], widened.pieces[1]])                          # dtypes differ
    with pytest.raises(TypeError):
        ShardedHostSlab([ps[0], HostSlab(torch.rand(3, 4, 3).half(), "cuda:0")])    # H differs
    with pytest.raises(TypeError):
        ShardedHostSlab([ps[0], HostSlab(torch.rand(2, 4, 5).half(), "cuda:0")])    # C differs
    with pytest.raises(TypeError):
        ShardedSlab(ps)                                                      # host pieces are not device pieces


@pytest.mark.parametrize("N,shards,gpus,ndev,device", [(1003, 2, None, 1, "cuda:0"), (1003, 3, 2, 4, "cuda:1"),
                                                       (7, 5, None, 8, "cuda:0"), (5, 8, None, 2, "cuda:0"),
                                                       (100, None, 3, 4, "cuda:2")])
def test_load_host_pieces_follow_load_sharded_on_one_memory_map(tmp_path, monkeypatch, N, shards, gpus, ndev, device):
    from coda_b200.datasets import Dataset, ShardedHostSlab, _load_plan, load_host, piece_plan
    from coda_b200.synth import shard_range
    H, C = 3, 7
    p, t = _slab_file(tmp_path, H, N, C, torch.bfloat16)
    _gpus(monkeypatch, [0] * ndev)
    for keep in (False, True):
        s = load_host(p, device, keep, shards=shards, gpus=gpus, chunk_items=64)
        assert isinstance(s, ShardedHostSlab) and s.shape == t.shape
        assert s.dtype == (torch.bfloat16 if keep else torch.float32)
        k = max(1, min(shards or gpus, N))
        want = piece_plan(N, k, gpus or min(k, ndev), torch.device(device).index, ndev)
        assert want == _load_plan(N, torch.device(device), shards, gpus)      # what load_sharded allocates from
        assert [(off, off + int(q.shape[1]), q.device.index) for q, off in s.layout()] == want
        assert [(lo, hi) for lo, hi, _ in want] == [shard_range(N, r, k) for r in range(k)]
        base = s.pieces[0].host
        for q, off in s.layout():                                              # views of one map: no host copy
            assert q.host.untyped_storage().data_ptr() == base.untyped_storage().data_ptr()
            assert q.host.data_ptr() == base.data_ptr() + off * C * 2
            assert torch.equal(q.host, t[:, off:off + int(q.shape[1])])
            assert q.chunk_items == min(64, (int(q.shape[1]) + 31) // 32 * 32)
    ds = Dataset(p, device, host=True, shards=shards, gpus=gpus)
    assert isinstance(ds.preds, ShardedHostSlab) and ds.preds.offsets == s.offsets
    one = Dataset(p, device, host=True).preds
    assert type(one).__name__ == "HostSlab"


# ---------------------------------------------------------------------------------------------------------------------
# refusals that need no device
# ---------------------------------------------------------------------------------------------------------------------
class _World2:
    world, rank = 2, 0


def test_refusals_on_host_pieces():
    from coda.options import LOSS_FNS
    from coda_b200 import CODA, IID, ModelPicker, ShardedHostSlab, TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    _, ps = _host_pieces()
    s = ShardedHostSlab(ps)
    ds = TensorDataset(s, torch.zeros(12, dtype=torch.int64))
    makers = (lambda **kw: CODA(ds, **kw), lambda **kw: IID(ds, LOSS_FNS["acc"], **kw),
              lambda **kw: ModelPicker(ds, **kw))
    for make in makers:
        for kw in ({"shards": 2}, {"gpus": 2}, {"shards": 4}, {"shards": 3, "gpus": 1}):
            with pytest.raises(ValueError, match="disagrees"):
                make(**kw)
        with pytest.raises(ValueError, match="torch.distributed"):
            make(comm=_World2())
    with pytest.raises(NotImplementedError, match="recompute_all"):
        CODA(ds, mode="recompute_all")
    with pytest.raises(NotImplementedError, match="ShardedHostSlab"):
        modelpicker_eps_search(ds, [0.5], iterations=1, pool_size=4, budget=2, seed=0)
