"""ModelPicker's epsilon search over every slab layout and over several runner GPUs (coda_b200.eps_search.hard_labels,
coda_b200_pool_gather): the search on a layout's HardLabels gives the bits of the search on the plain device tensor of
the same slab (a compact layout: of the whole CompactSlab) for any runner count and block size; the gather equals torch
indexing; device memory comes back; the command line's --gpus route writes what the plain route writes."""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
KEYS = ("picks", "best", "pick_tie", "best_tie", "pool_accuracies", "labels")


def _cuts(N, k):
    return [(N * r // k, N * (r + 1) // k) for r in range(k)]


def _same(a, b):
    for k in KEYS:
        assert np.array_equal(a[k], b[k]), k
    assert a["metrics"] == b["metrics"]
    assert (a["best_avg"], a["best_fast"]) == (b["best_avg"], b["best_fast"])


def _search(data, pools, **kw):
    from coda_b200.eps_search import modelpicker_eps_search
    return modelpicker_eps_search(data, epsilons=(0.35, 0.46), budget=kw.pop("budget", 20), seed=5,
                                  realisations=pools, **kw)


def _dense_layouts(preds):
    """``preds`` (CPU, at its dtype) as a ShardedSlab of 3 pieces, a HostSlab scanned in 32-item chunks and a
    ShardedHostSlab of 2 pieces, all on this GPU."""
    from coda_b200 import HostDataset, HostSlab, ShardedHostSlab, ShardedSlab, TensorDataset
    N = preds.shape[1]
    yield "sharded3", TensorDataset(ShardedSlab([preds[:, lo:hi].contiguous().to(DEV) for lo, hi in _cuts(N, 3)]))
    yield "host", HostDataset(HostSlab(preds, DEV, chunk_items=32))
    yield "host_pieces2", TensorDataset(ShardedHostSlab([HostSlab(preds[:, lo:hi], DEV, chunk_items=32)
                                                          for lo, hi in _cuts(N, 2)]))


@pytest.mark.parametrize("H,C", [(1, 2), (5, 10), (64, 10), (256, 100), (1024, 2)])
def test_every_layout_gives_the_plain_search(H, C):
    from coda_b200 import CompactDataset, CompactSlab, ShardedCompactSlab, TensorDataset
    from coda_b200.eps_search import hard_labels
    from coda_b200.synth import synth
    N, P = 301, 150                                        # N not a multiple of 32; P above a third of N
    preds, _ = synth(H, N, C, seed=H + C)
    pools = np.stack([np.random.default_rng(r).permutation(N)[:P] for r in range(3)])
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        p = preds.to(dtype)
        ref = _search(TensorDataset(p.to(DEV)), pools)
        for name, ds in _dense_layouts(p):
            got = _search(hard_labels(ds), pools)
            _same(got, ref)
        _same(_search(hard_labels(TensorDataset(p.to(DEV))), pools, gpus=1), ref)
    whole = CompactSlab.from_dense(preds.to(DEV), min(4, C - 1))
    ref = _search(CompactDataset(whole), pools)
    pieces = ShardedCompactSlab([whole.narrow_items(lo, hi) for lo, hi in _cuts(N, 3)])
    _same(_search(hard_labels(CompactDataset(pieces)), pools), ref)


def test_runner_blocks_and_budgets(monkeypatch):
    """R = 1, R not a multiple of the runners, and blocks of one and two realisations per runner."""
    from coda_b200 import ShardedSlab, TensorDataset
    from coda_b200 import eps_search
    from coda_b200.synth import synth
    H, N, C, P = 24, 203, 6, 90
    preds, _ = synth(H, N, C, seed=3)
    pools = np.stack([np.random.default_rng(10 + r).permutation(N)[:P] for r in range(7)])
    ref = _search(TensorDataset(preds.to(DEV)), pools, budget=P)
    table = eps_search.hard_labels(TensorDataset(ShardedSlab([preds[:, lo:hi].contiguous().to(DEV)
                                                              for lo, hi in _cuts(N, 3)])))
    for per_block in (1, 2):
        monkeypatch.setattr(eps_search, "POOL_TABLE_BYTES", per_block * P * (2 * H + 9))
        _same(_search(table, pools, budget=P), ref)
        _same(_search(table, pools[4:5], budget=P), _search(TensorDataset(preds.to(DEV)), pools[4:5], budget=P))
        if torch.cuda.device_count() >= 2:
            _same(_search(table, pools, budget=P, gpus=2), ref)
            _same(_search(table, pools[:1], budget=P, gpus=2), _search(table, pools[:1], budget=P))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_pieces_on_two_gpus():
    from coda_b200 import ShardedHostSlab, HostSlab, ShardedSlab, TensorDataset
    from coda_b200.eps_search import hard_labels
    from coda_b200.synth import synth
    H, N, C = 40, 257, 8
    preds, _ = synth(H, N, C, seed=4)
    pools = np.stack([np.random.default_rng(r).permutation(N)[:140] for r in range(5)])
    ref = _search(TensorDataset(preds.to(DEV)), pools)
    devs = [torch.device("cuda", d) for d in (0, 1)]
    for ds in (TensorDataset(ShardedSlab([preds[:, lo:hi].contiguous().to(d) for (lo, hi), d in zip(_cuts(N, 2), devs)])),
               TensorDataset(ShardedHostSlab([HostSlab(preds[:, lo:hi], d, chunk_items=64)
                                              for (lo, hi), d in zip(_cuts(N, 2), devs)]))):
        table = hard_labels(ds)
        assert table.devices == [0, 1]
        for gpus in (None, 1, 2):
            _same(_search(table, pools, gpus=gpus), ref)


def test_given_labels_on_pieces():
    from coda_b200 import HostSlab, ShardedHostSlab, TensorDataset
    from coda_b200.eps_search import hard_labels
    from coda_b200.synth import synth
    H, N, C = 16, 190, 7
    preds, labels = synth(H, N, C, seed=6)
    pools = np.stack([np.random.default_rng(r).permutation(N)[:120] for r in range(4)])
    ref = _search(TensorDataset(preds.to(DEV)), pools, labels=labels)
    assert np.array_equal(ref["labels"], labels.numpy())
    table = hard_labels(TensorDataset(ShardedHostSlab([HostSlab(preds[:, lo:hi], DEV) for lo, hi in _cuts(N, 3)])))
    _same(_search(table, pools, labels=labels), ref)
    _same(_search(table, pools, labels=labels.to(DEV)), ref)


@pytest.mark.parametrize("H", [1, 6, 12, 64, 1023])
def test_pool_gather_equals_torch_indexing(H):
    """One call at a time: slots anywhere in a larger output, a piece that holds no pair, every vector width."""
    from coda_b200 import _native as nat
    lib = nat.load()
    g = torch.Generator().manual_seed(H)
    N, K, M = 97, 150, 400
    hard = torch.randint(-32768, 32767, (N, H), generator=g, dtype=torch.int16).to(DEV)
    dis = torch.randint(0, 2, (N,), generator=g, dtype=torch.uint8).to(DEV)
    lab = torch.randint(0, 1 << 40, (N,), generator=g, dtype=torch.int64).to(DEV)
    items = torch.randint(0, N, (K,), generator=g).to(DEV)
    slots = torch.randperm(M, generator=g)[:K].to(DEV)
    oh = torch.full((M, H), 7, dtype=torch.int16, device=DEV)
    od = torch.full((M,), 3, dtype=torch.uint8, device=DEV)
    ol = torch.full((M,), -1, dtype=torch.int64, device=DEV)
    s = torch.cuda.current_stream(DEV).cuda_stream
    p = lambda t: t.data_ptr()
    nat.check(lib.coda_b200_pool_gather(p(hard), p(dis), p(lab), H, p(slots), p(items), K, p(oh), p(od), p(ol), s))
    wh, wd, wl = (torch.full_like(oh, 7), torch.full_like(od, 3), torch.full_like(ol, -1))
    wh[slots], wd[slots], wl[slots] = hard[items], dis[items], lab[items]
    assert torch.equal(oh, wh) and torch.equal(od, wd) and torch.equal(ol, wl)
    nat.check(lib.coda_b200_pool_gather(p(hard), p(dis), p(lab), H, None, None, 0, p(oh), p(od), p(ol), s))
    torch.cuda.synchronize()
    assert torch.equal(oh, wh) and torch.equal(od, wd) and torch.equal(ol, wl)


def test_device_memory_comes_back_and_the_slab_can_go():
    from coda_b200 import HostSlab, ShardedSlab, TensorDataset
    from coda_b200.eps_search import hard_labels
    from coda_b200.synth import synth
    H, N, C = 32, 300, 10
    preds, _ = synth(H, N, C, seed=8)
    pools = np.stack([np.random.default_rng(r).permutation(N)[:100] for r in range(3)])
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(DEV)
    ds = TensorDataset(ShardedSlab([preds[:, lo:hi].contiguous().to(DEV) for lo, hi in _cuts(N, 2)]))
    table = hard_labels(ds)
    del ds                                                 # the table holds no reference to the slab
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) - before < preds.numel() * 4 // 10
    res = _search(table, pools)
    del table
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) == before
    _search(TensorDataset(preds.to(DEV)), pools)           # the plain route drops its table too
    _search(hard_labels(TensorDataset(HostSlab(preds, DEV))), pools)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) == before
    assert res["picks"].shape == (2, 3, 20)


def test_bad_scores_raise_as_the_selectors_raise():
    from coda_b200 import HostSlab, ShardedSlab, TensorDataset
    from coda_b200.eps_search import hard_labels
    from coda_b200.synth import synth
    preds, _ = synth(6, 100, 4, seed=9)
    bad = preds.clone()
    bad[2, 70, 1] = float("nan")
    with pytest.raises(RuntimeError, match="NaN"):
        hard_labels(TensorDataset(HostSlab(bad, DEV, chunk_items=32)))
    bad = preds.clone()
    bad[1, 10, 0] = 3.0
    with pytest.raises(ValueError, match=r"\[0, 1\]"):
        hard_labels(TensorDataset(ShardedSlab([bad[:, :50].contiguous().to(DEV), bad[:, 50:].contiguous().to(DEV)])))


@pytest.mark.parametrize("kind", ["fp16", "compact"])
def test_cli_gpus_1_writes_the_plain_entry(kind, tmp_path, monkeypatch):
    from coda_b200 import CompactSlab
    from coda_b200.eps_search import main
    from coda_b200.synth import synth
    preds, _ = synth(20, 230, 6, seed=11)
    path = tmp_path / "task.pt"
    if kind == "fp16":
        torch.save(preds.half(), path)
    else:
        CompactSlab.from_dense(preds.to(DEV), 3).save(str(path))
    args = ["--preds", str(path), "--epsilons", "0.36,0.42,0.47", "--iterations", "6", "--pool-size", "80",
            "--budget", "30", "--threshold", "0.5", "--seed", "3"]
    out = {}
    for name, extra in (("plain", []), ("gpus", ["--gpus", "1"])):
        d = tmp_path / name
        d.mkdir()
        monkeypatch.chdir(d)
        assert main(args + extra) == 0
        out[name] = json.loads((d / "best_epsilons.json").read_text())
    assert out["gpus"] == out["plain"] and list(out["plain"]) == ["task.pt"]


def test_a_round_stages_every_runner_before_any_run_waits():
    """Two runners (both on this GPU) whose blocks read the same piece.  Staging the second runner's block -- its index
    uploads block the host until the piece's stream is idle -- must not wait for the first runner's runs: every block
    is staged before any block's runs are launched.  The host is back long before the runs end, and the blocks hold
    the plain search's bits."""
    import time
    from coda_b200 import TensorDataset, _native as nat
    from coda_b200 import eps_search
    from coda_b200.synth import synth
    H, N, C, P, B = 64, 2000, 10, 600, 300
    eps = (0.35, 0.37, 0.39, 0.41, 0.43, 0.45, 0.47, 0.49)
    preds, _ = synth(H, N, C, seed=12)
    preds = preds.to(DEV)
    pools = np.stack([np.random.default_rng(20 + r).permutation(N)[:P] for r in range(2)])
    ref = eps_search.modelpicker_eps_search(TensorDataset(preds), epsilons=eps, budget=B, seed=9, realisations=pools)
    lib = nat.load()
    table = eps_search.hard_labels(TensorDataset(preds))
    gammas = np.array([np.float32((1.0 - e) / e) for e in eps], dtype=np.float32)
    keys = np.array([[eps_search.eps_search_run_key(9, e, r) for r in range(2)] for e in range(len(eps))],
                    dtype=np.uint64)
    labs = eps_search._piece_labels(lib, table, None)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    staged = eps_search._enqueue_round(lib, table, labs, [(DEV, pools[r:r + 1], keys[:, r:r + 1]) for r in range(2)],
                                       gammas, B)
    t_enqueue = time.perf_counter() - t0
    busy = not torch.cuda.current_stream(DEV).query()
    torch.cuda.synchronize()
    t_all = time.perf_counter() - t0
    assert busy and t_enqueue < 0.25 * t_all, (t_enqueue, t_all)
    for r, b in enumerate(staged):
        for k in ("picks", "best", "pick_tie", "best_tie"):
            assert np.array_equal(b[k].cpu().numpy()[:, 0], ref[k][:, r]), (r, k)
        assert np.array_equal(b["acc"].cpu().numpy()[0], ref["pool_accuracies"][r])
