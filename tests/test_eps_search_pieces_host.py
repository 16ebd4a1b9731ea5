"""CPU tests of the epsilon search over pieces (coda_b200.eps_search): the realisation split into runner blocks, the pool
table's local indices against a NumPy model of gather and concatenation, the command line's --gpus route with stand-ins,
the refusal that points at hard_labels, and the gather entry point of the C ABI."""
import os
import re

import numpy as np
import pytest
import torch

from helpers import ROOT


@pytest.mark.parametrize("R,runners,per_block", [(1, 1, 1), (1, 3, 5), (7, 2, 3), (10, 4, 1), (1000, 8, 97),
                                                 (5, 5, 100), (3, 8, 2)])
def test_realisation_blocks_take_every_realisation_once_in_order(R, runners, per_block):
    from coda_b200.eps_search import realisation_blocks
    blocks = realisation_blocks(R, runners, per_block)
    assert len(blocks) == runners
    flat = [r for b in blocks for r0, r1 in b for r in range(r0, r1)]
    assert flat == list(range(R))
    for b in blocks:
        assert all(0 < r1 - r0 <= per_block for r0, r1 in b)
        assert all(b[i][1] == b[i + 1][0] for i in range(len(b) - 1))     # one contiguous range per runner
    sizes = [sum(r1 - r0 for r0, r1 in b) for b in blocks]
    assert max(sizes) - min(sizes) <= 1


@pytest.mark.parametrize("cuts", [[0], [0, 100], [0, 37, 38, 290], [0, 150, 151]])
def test_pool_table_indexes_the_concatenated_gathers(cuts):
    """Each piece gathers the rows of its items in pool-major order; the runner's table is their concatenation; the local
    pool must name the row of the same item there."""
    from coda_b200.eps_search import pool_table
    rng = np.random.default_rng(len(cuts))
    N, H = 301, 7
    hard = rng.integers(0, 50, size=(N, H))
    pools = np.stack([rng.permutation(N)[:160] for _ in range(5)])
    pools[2, :5] = pools[0, :5]                                           # an item in two realisations
    local, items = pool_table(pools, cuts)
    assert local.shape == pools.shape and len(items) == len(cuts)
    ends = cuts[1:] + [N]
    table = np.concatenate([hard[lo:hi][it] for lo, hi, it in zip(cuts, ends, items)])
    assert table.shape == (pools.size, H)
    assert np.array_equal(table[local], hard[pools])
    assert sorted(local.reshape(-1).tolist()) == list(range(pools.size))
    for lo, hi, it in zip(cuts, ends, items):
        want = pools.reshape(-1)[(pools.reshape(-1) >= lo) & (pools.reshape(-1) < hi)] - lo
        assert np.array_equal(it, want)                                   # pool-major order within a piece
    empty = pool_table(np.array([[0, 1, 2]]), [0, 100])[1]
    assert empty[1].size == 0                                             # a piece that holds no pool item


def _fake_search(calls):
    def search(data, **kw):
        calls.append((data, kw))
        m = {e: {"success_mean": [1.0], "acc_mean": [1.0], "avg_success": 1.0, "fastest_t": 0} for e in kw["epsilons"]}
        return {"best_avg": kw["epsilons"][0], "best_fast": kw["epsilons"][-1], "metrics": m}
    return search


def test_cli_gpus_route_loads_a_table_and_passes_gpus(tmp_path, monkeypatch):
    import json
    from coda_b200 import eps_search
    from coda_b200.synth import synth
    preds, _ = synth(4, 30, 3, seed=1)
    path = tmp_path / "taskA.pt"
    torch.save(preds, path)
    monkeypatch.chdir(tmp_path)
    tables = []
    monkeypatch.setattr(eps_search, "_table_from_file",
                        lambda p, dev, gpus: tables.append((p, gpus)) or ("table", p, gpus))
    calls = []
    args = ["--preds", str(path), "--epsilons", "0.4,0.45", "--iterations", "3", "--seed", "2"]
    assert eps_search.main(args + ["--gpus", "2"], search=_fake_search(calls)) == 0
    assert tables == [(str(path), 2)]
    data, kw = calls[0]
    assert data == ("table", str(path), 2) and kw["gpus"] == 2 and kw["iterations"] == 3 and kw["seed"] == 2
    assert json.loads((tmp_path / "best_epsilons.json").read_text()) == {"taskA.pt": {"best_avg": 0.4,
                                                                                     "best_fast": 0.45}}
    # too large for the device, no --gpus: the table route on one GPU, and today's keywords
    os.remove(tmp_path / "best_epsilons.json")
    monkeypatch.setattr(eps_search, "_auto_pieces", lambda p, dev: 1)
    assert eps_search.main(args, search=_fake_search(calls)) == 0
    assert tables[-1] == (str(path), 1) and calls[-1][0] == ("table", str(path), 1)
    assert "gpus" not in calls[-1][1]
    # it fits: the plain load, as before
    os.remove(tmp_path / "best_epsilons.json")
    monkeypatch.setattr(eps_search, "_auto_pieces", lambda p, dev: None)
    assert eps_search.main(args, search=_fake_search(calls)) == 0
    assert len(tables) == 2 and tuple(calls[-1][0].preds.shape) == (4, 30, 3) and "gpus" not in calls[-1][1]


def test_cli_route_without_gpus_follows_the_file_and_free_memory(tmp_path, monkeypatch):
    """A dense file too large for the device: one host-resident piece; a compact file too large: compact pieces over
    every visible GPU, or the plain load with one GPU (a compact slab has no host-resident form); a file that fits or in
    torch's legacy format: the plain load."""
    from coda_b200 import CompactSlab, datasets
    from coda_b200.eps_search import _auto_pieces
    dense = tmp_path / "dense.pt"
    torch.save(torch.full((2, 10, 3), 1 / 3), dense)                          # 240 bytes as fp32
    legacy = tmp_path / "legacy.pt"
    torch.save(torch.full((2, 10, 3), 1 / 3), legacy, _use_new_zipfile_serialization=False)
    compact = tmp_path / "compact.pt"
    CompactSlab(torch.zeros((2, 10, 1), dtype=torch.int16), torch.ones((2, 10, 1)), 3).save(str(compact))   # 120
    cuda = torch.device("cuda", 0)
    assert _auto_pieces(str(dense), torch.device("cpu")) is None
    for free, gpus, want in ((1000, 1, (None, None, None)), (200, 1, (1, None, None)), (200, 4, (1, None, None)),
                             (100, 1, (1, None, None)), (100, 3, (1, 3, None))):
        monkeypatch.setattr(datasets, "_free_bytes", lambda index: free)
        monkeypatch.setattr(torch.cuda, "device_count", lambda: gpus)
        assert tuple(_auto_pieces(str(p), cuda) for p in (dense, compact, legacy)) == want, (free, gpus)


def test_cli_refuses_more_gpus_than_visible(tmp_path):
    from coda_b200.eps_search import _table_from_file
    with pytest.raises(ValueError, match="GPUs are visible"):
        _table_from_file(str(tmp_path / "x.pt"), torch.device("cpu"), torch.cuda.device_count() + 1)


def test_a_sharded_slab_is_refused_with_the_route_that_takes_it():
    from coda_b200 import ShardedSlab, TensorDataset
    from coda_b200.eps_search import modelpicker_eps_search
    s = ShardedSlab([torch.full((2, 3, 4), 0.25), torch.full((2, 5, 4), 0.25)])
    with pytest.raises(NotImplementedError, match=r"ShardedSlab.*hard_labels\(dataset\)"):
        modelpicker_eps_search(TensorDataset(s, None))


def test_pool_gather_is_declared_and_bound():
    from coda_b200 import _native as nat
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    m = re.search(r"\bcoda_b200_pool_gather\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
    assert m and len(m.group(1).split(",")) == 11
    assert len(nat.SIGNATURES["coda_b200_pool_gather"][1]) == 11
    assert nat.VERSION == 203
    assert hasattr(nat.load(), "coda_b200_pool_gather")
