"""The competing selectors on N-range shards (in-process shards on one or more GPUs, one process per GPU) and on the
compact slab.  Host mirrors of the three cross-shard merges run on the CPU; everything else on the GPU: sharded runs
against the reference goldens, against one shard, and the compact slab against its densified twin."""
import hashlib
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from helpers import GOLDEN, ROOT

METHODS = ["iid", "uncertainty", "activetesting", "vma", "model_picker"]


def _digest(b):
    return int.from_bytes(hashlib.sha256(b).digest()[:8], "little", signed=True)


def _rng_digests():
    d = [_digest(repr(random.getstate()).encode()), _digest(torch.get_rng_state().numpy().tobytes())]
    if torch.cuda.is_available():
        d.append(_digest(torch.cuda.get_rng_state().numpy().tobytes()))
    return tuple(d)


def _seed_all():
    random.seed(0)
    np.random.seed(0)
    torch.manual_seed(0)


# ------------------------------------------------------------------------------------------------------------------
# CPU: host mirrors of the merges (coda_b200.dist) against one evaluation over the whole vector
# ------------------------------------------------------------------------------------------------------------------
def _splits(rng, n, world):
    """Random contiguous cuts of [0, n) into `world` ranges, empty ranges allowed."""
    cuts = np.sort(rng.integers(0, n + 1, size=world - 1))
    b = [0, *cuts.tolist(), n]
    return [(b[r], b[r + 1]) for r in range(world)]


def _extreme_rec(v, unl, want_max):
    """(value, count) of one shard's unlabeled items: the per-shard record of select_extreme."""
    vals = v[unl]
    if not len(vals):
        return 0.0, 0
    best = vals.max() if want_max else vals.min()
    return float(best), int((vals == best).sum())


@pytest.mark.parametrize("want_max", [False, True])
def test_extreme_and_kth_merge_mirror_one_vector(want_max):
    from coda_b200.dist import kth_owner, merge_extreme
    rng = np.random.default_rng(3)
    for trial in range(300):
        n = int(rng.integers(1, 60))
        world = int(rng.integers(1, 7))
        v = rng.choice(np.array([0.5, 1.0, 2.0, np.inf], np.float32), size=n)
        unl = rng.random(n) < 0.7
        if trial % 5 == 0:
            lo, hi = _splits(rng, n, 2)[0]
            unl[lo:hi] = False                                    # an all-labeled range
        cuts = _splits(rng, n, world)
        recs = [_extreme_rec(v[lo:hi], unl[lo:hi], want_max) for lo, hi in cuts]
        whole = _extreme_rec(v, unl, want_max)
        for r in range(world):
            val, cnt, lower, mine = merge_extreme(recs, want_max, r)
            assert (cnt, val if cnt else 0.0) == (whole[1], whole[0] if whole[1] else 0.0)
            lo, hi = cuts[r]
            assert lower == int(((v[:lo] == whole[0]) & unl[:lo]).sum()) if cnt else lower == 0
            assert mine == (int(((v[lo:hi] == whole[0]) & unl[lo:hi]).sum()) if cnt else 0)
        tied = np.nonzero((v == whole[0]) & unl)[0] if whole[1] else []
        for k, item in enumerate(tied):
            owner, kk = kth_owner(recs, want_max, k)
            lo, hi = cuts[owner]
            local = np.nonzero((v[lo:hi] == whole[0]) & unl[lo:hi])[0]
            assert lo + local[kk] == item
        assert kth_owner(recs, want_max, len(tied)) == (-1, -1)


def test_weighted_draw_owner_and_position_mirror_one_vector():
    """Integer weights (exact fp64 sums in any association): owner, its base and the global position give the item that
    bisect_right over the cumulative weights of the whole vector gives, for every target including the ends."""
    from coda_b200.dist import draw_owner
    rng = np.random.default_rng(5)
    for trial in range(300):
        n = int(rng.integers(1, 50))
        world = int(rng.integers(1, 7))
        w = rng.integers(0, 4, size=n).astype(np.float64)
        unl = rng.random(n) < 0.75
        if trial % 4 == 0:
            lo, hi = _splits(rng, n, 2)[0]
            unl[lo:hi] = False
        if not unl.any():
            unl[int(rng.integers(0, n))] = True
        items = np.nonzero(unl)[0]
        cum = np.cumsum(w[items])
        total = float(cum[-1])
        cuts = _splits(rng, n, world)
        sums = [float(w[lo:hi][unl[lo:hi]].sum()) for lo, hi in cuts]
        counts = [int(unl[lo:hi].sum()) for lo, hi in cuts]
        for u in [0.0, *rng.random(8).tolist(), 1.0 - 2 ** -53]:
            owner, base, pos, target = draw_owner(sums, counts, u)
            assert target == u * total
            lo, hi = cuts[owner]
            assert counts[owner] > 0 and pos == sum(counts[:owner]) and base == sum(sums[:owner])
            # the owner's in-chunk walk from (base, pos)
            c, p, pick = base, pos, None
            for i in np.nonzero(unl[lo:hi])[0]:
                c += w[lo + i]
                if c > target:
                    pick = (p, lo + i)
                    break
                last = (p, lo + i)
                p += 1
            pick = pick or last
            j = int(np.searchsorted(cum, target, side="right"))
            j = min(j, len(items) - 1)                             # at or beyond the total: the last item
            assert pick == (j, int(items[j])), (trial, u)


def test_compact_item_column_is_the_densified_column():
    from coda_b200 import CompactSlab
    from coda_b200.synth import synth_compact
    ids, probs, _ = synth_compact(7, 90, 23, 3, seed=4)
    slab = CompactSlab(ids, probs, 23)
    dense = slab.densify()
    for i in (0, 1, 44, 89):
        assert torch.equal(slab.item_column(i), dense[:, i])


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def _make(method, ds, **kw):
    from coda.options import LOSS_FNS
    from coda_b200 import IID, VMA, ActiveTesting, ModelPicker, Uncertainty
    if method == "model_picker":
        return ModelPicker(ds, **kw)
    return {"iid": IID, "uncertainty": Uncertainty, "activetesting": ActiveTesting, "vma": VMA}[method](
        ds, LOSS_FNS["acc"], **kw)


def _trace(sel, labels, steps, entropies=False):
    """(idx, q, best, RNG digests[, entropy digest]) per step of main.py's loop."""
    out = [(None, None, int(sel.get_best_model_prediction()), _rng_digests())]
    for _ in range(steps):
        idx, q = sel.get_next_item_to_label()
        ent = _digest(sel.entropies.cpu().numpy().tobytes()) if entropies else None
        sel.add_label(idx, int(labels[idx]), q)
        out.append((idx, q, int(sel.get_best_model_prediction()), _rng_digests(), ent))
    return out


def _golden_cases(method):
    names = sorted(f[:-4] for f in os.listdir(GOLDEN) if f.startswith(f"baseline_{method}_h") and f.endswith(".npz"))
    assert names, method
    return names


@pytest.mark.gpu
@pytest.mark.parametrize("shards", [2, 3])
@pytest.mark.parametrize("method", ["iid", "activetesting", "vma"])
def test_sharded_stochastic_baselines_follow_the_reference_draw_for_draw(method, shards):
    from coda_b200 import TensorDataset
    from coda_b200.synth import synth
    for name in _golden_cases(method):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        g = {k: z[k] for k in z.files}
        preds, labels = synth(int(g["H"]), int(g["N"]), int(g["C"]), int(g["data_seed"]))
        _seed_all()
        sel = _make(method, TensorDataset(preds.cuda(), labels.cuda()), shards=shards)
        assert len(sel.states) == shards and sel.group.world == shards
        if "score" in g:
            np.testing.assert_allclose(sel.score.cpu().numpy(), g["score"], rtol=1e-5, atol=1e-6)
        assert int(sel.get_best_model_prediction()) == int(g["best0"])
        for k in range(int(g["steps"])):
            idx, q = sel.get_next_item_to_label()
            assert isinstance(idx, int) and idx == int(g["idx"][k]), (name, k, idx, int(g["idx"][k]))
            np.testing.assert_allclose(q, g["q"][k], rtol=1e-5)
            sel.add_label(idx, int(labels[idx]), q)
            best = sel.get_best_model_prediction()
            assert isinstance(best, torch.Tensor) and best.dim() == 0 and int(best) == int(g["best"][k]), (name, k)
            assert _rng_digests()[:2] == (int(g["py"][k]), int(g["torch"][k])), (name, k)
            if "lure" in g:
                np.testing.assert_allclose(sel.get_risk_estimates().cpu().numpy(), g["lure"][k], atol=1e-6)
        assert all(int(st.flags.item()) == 0 for st in sel.states)
        sel.close()


@pytest.mark.gpu
@pytest.mark.parametrize("shards", [2, 3])
@pytest.mark.parametrize("method", ["uncertainty", "model_picker"])
def test_sharded_arg_extreme_baselines_follow_the_reference(method, shards):
    """Uncertainty / ModelPicker on shards: the same steps as one shard (bit-identical scores), and the reference's picks
    until its own best and runner-up are within fp32 noise."""
    from coda_b200 import TensorDataset
    from coda_b200.synth import synth
    for name in _golden_cases(method):
        z = np.load(os.path.join(GOLDEN, name + ".npz"))
        g = {k: z[k] for k in z.files}
        preds, labels = synth(int(g["H"]), int(g["N"]), int(g["C"]), int(g["data_seed"]))
        runs = []
        for s in (1, shards):
            _seed_all()
            sel = _make(method, TensorDataset(preds.cuda(), labels.cuda()), shards=s)
            if method == "uncertainty":
                assert np.allclose(sel.score.cpu().numpy(), g["score"], atol=1e-6)
                runs.append((sel.score.cpu().numpy(), _trace(sel, labels, int(g["steps"]))))
            else:
                runs.append((None, _trace(sel, labels, int(g["steps"]), entropies=True)))
            sel.close()
        if method == "uncertainty":
            assert np.array_equal(runs[0][0], runs[1][0])
        assert runs[0][1] == runs[1][1], name                      # picks, q, best models, RNG, entropy bits
        trace = runs[1][1][1:]
        for k, (idx, q, best, dig, _e) in enumerate(trace):
            if method == "uncertainty":
                score = g["score"].copy()
                score[[t[0] for t in trace[:k]]] = -np.inf
                top2 = np.sort(score)[-2:]
                if top2[1] - top2[0] <= 1e-6:
                    break
                assert idx == int(g["idx"][k]) and best == int(g["best"][k]) and dig[:2] == (int(g["py"][k]), int(g["torch"][k]))
            else:
                ref = g["ent"][k]
                m = np.nanmin(ref)
                tol = int(g["C"]) * float(np.spacing(np.float32(np.nanmax(ref[np.isfinite(ref)])))) / 2 + 1e-6
                if np.sum(ref <= m + tol) > 1:
                    assert ref[idx] <= m + tol
                    break
                assert idx == int(g["idx"][k]) and dig[1] == int(g["torch"][k]), (name, k)


@pytest.mark.gpu
@pytest.mark.parametrize("dense", [False, True])
@pytest.mark.parametrize("method", METHODS)
def test_shard_counts_give_the_same_run(method, dense):
    """synth(32, 50 000, 10) for 30 steps on 1, 2, 3 and 5 shards of one GPU: the same picks, q bits, best models and
    RNG states; static scores and ModelPicker entropies bit-identical to one shard."""
    from coda_b200 import TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(32, 50_000, 10, 11, dense=dense)
    preds, lab_dev = preds.cuda(), labels.cuda()
    ref = None
    for shards in (1, 2, 3, 5):
        _seed_all()
        sel = _make(method, TensorDataset(preds, lab_dev), shards=shards)
        assert len(sel.states) == shards
        score = sel.score.cpu() if method in ("uncertainty", "activetesting", "vma") else None
        run = (score, _trace(sel, labels, 30, entropies=method == "model_picker"))
        assert all(int(st.flags.item()) == 0 for st in sel.states)
        assert int(sum(int(st.labeled.sum()) for st in sel.states)) == 30
        sel.close()
        if ref is None:
            ref = run
            continue
        if score is not None:
            assert torch.equal(run[0], ref[0]), shards
        assert run[1] == ref[1], shards


def _compact_case(H, N, C, K, seed):
    from coda_b200 import CompactSlab
    from coda_b200.synth import synth_compact
    ids, probs, labels = synth_compact(H, N, C, K, seed=seed)
    return CompactSlab(ids, probs, C).to(torch.device("cuda:0")), labels


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("shape", [(24, 1200, 30, 4, 3), (40, 700, 150, 3, 5), (9, 500, 8, 2, 7)])
def test_compact_slab_against_its_densified_twin(method, shape):
    """The selectors on a compact slab and on TensorDataset(slab.densify()): identical hard / disagree, ensemble-derived
    scores within 1e-6 relative, identical picks while the best and runner-up are further apart than that; and the
    compact slab on 2 shards equals one shard (bit-identical scores)."""
    from coda_b200 import CompactDataset, TensorDataset
    H, N, C, K, seed = shape
    slab, labels = _compact_case(H, N, C, K, seed)
    dense = slab.densify()
    _seed_all()
    sel = _make(method, CompactDataset(slab, labels.cuda()))
    _seed_all()
    twin = _make(method, TensorDataset(dense, labels.cuda()))
    for st, tw in ((sel.state, twin.state), ):
        h1, d1, e1 = st.scan(ens=True)
        h2, d2, e2 = tw.scan(ens=True)
        assert torch.equal(h1, h2) and torch.equal(d1, d2)
        np.testing.assert_allclose(e1.cpu().numpy(), e2.cpu().numpy(), rtol=1e-6, atol=1e-6)
    if method in ("uncertainty", "activetesting", "vma"):
        np.testing.assert_allclose(sel.score.cpu().numpy(), twin.score.cpu().numpy(), rtol=1e-6, atol=1e-6)
    _seed_all()
    a = _trace(sel, labels, 20, entropies=method == "model_picker")
    _seed_all()
    b = _trace(twin, labels, 20, entropies=method == "model_picker")
    if method == "uncertainty":
        score = twin.score.cpu().numpy().copy()
        for k in range(20):
            top2 = np.sort(score)[-2:]
            if top2[1] - top2[0] <= 1e-6 * max(1.0, abs(float(top2[1]))):
                break
            assert a[k + 1][0] == b[k + 1][0], k
            score[b[k + 1][0]] = -np.inf
    else:
        assert [t[0] for t in a] == [t[0] for t in b]
        assert [t[2] for t in a] == [t[2] for t in b]
        if method in ("iid", "model_picker"):
            assert a == b
    score = sel.score.cpu() if method != "iid" and method != "model_picker" else None
    sel.close()
    twin.close()
    two = _make(method, CompactDataset(slab, labels.cuda()), shards=2)
    if score is not None:
        assert torch.equal(two.score.cpu(), score)
    _seed_all()
    assert _trace(two, labels, 20, entropies=method == "model_picker") == a
    assert all(int(st.flags.item()) == 0 for st in two.states)
    two.close()


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_main_py_driver_with_three_in_process_shards(tmp_path, method):
    """The main.py-style driver of test_baselines.py with CODA_B200_GPUS=3 (three shards, sharing a GPU on a 1-GPU box) reproduces the
    reference's run under that test's rules."""
    from test_baselines import _DRIVER          # also puts tests/golden on sys.path
    import make_cfg1_golden as mk1
    from coda_b200.synth import synth
    gall = json.load(open(os.path.join(GOLDEN, "baselines_main_py.json")))
    g, task, iters = gall["methods"][method], gall["task"], gall["iters"]
    d = str(tmp_path)
    preds, labels = synth(task["H"], task["N"], task["C"], task["seed"])
    torch.save(preds, os.path.join(d, task["name"] + ".pt"))
    torch.save(labels, os.path.join(d, task["name"] + "_labels.pt"))
    driver = _DRIVER.replace("    return selector.stochastic\n",
                             "    print('SHARDS', len(selector.states))\n    return selector.stochastic\n")
    with open(os.path.join(d, "driver.py"), "w") as f:
        f.write(driver)
    log = os.path.join(d, "mlflow.jsonl")
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests", "stubs")]),
               MLFLOW_STUB_LOG=log, PYTHONSAFEPATH="1", CODA_B200_GPUS="3")
    env.pop("CODA_REFERENCE_PATH", None)
    cmd = [sys.executable, os.path.join(d, "driver.py"), "--task", task["name"], "--data-dir", d, "--method", method,
           "--seeds", "1", "--iters", str(iters)]
    r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=d, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "SHARDS 3" in r.stdout
    out = mk1.parse_log(log)
    assert out["runs"] == g["runs"] and len(out["chosen_idx"]) == iters
    tol = {"uncertainty": 1e-6, "model_picker": 2e-6}.get(method)
    n = iters
    if tol is not None:
        n = next((k for k, gap in enumerate(g["gap"]) if gap <= tol), iters)
    assert out["chosen_idx"][:n] == g["chosen_idx"][:n], method
    assert out["true_class"][:n] == g["true_class"][:n]
    if method != "model_picker":
        assert out["best_model"][:n] == g["best_model"][:n]
        np.testing.assert_allclose(out["regret"][:n], g["regret"][:n], atol=1e-7)
        np.testing.assert_allclose(out["cumulative_regret"][:n], g["cumulative_regret"][:n], atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_two_gpus_in_one_process_equal_one_gpu(method):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from coda_b200 import TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(48, 30011, 14, 4)
    runs = []
    for gpus in (1, 2):
        _seed_all()
        sel = _make(method, TensorDataset(preds.cuda(0), labels.cuda(0)), gpus=gpus)
        assert len({st.dev for st in sel.states}) == gpus
        runs.append(_trace(sel, labels, 15, entropies=method == "model_picker"))
        sel.close()
    assert runs[0] == runs[1]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_equals_one_gpu(world):
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(29500 + world),
           os.path.join(ROOT, "tests", "baselines_mgpu_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("BASELINES_MGPU ")][-1]
    res = json.loads(line[len("BASELINES_MGPU "):])
    for method, o in res.items():
        assert o["same_on_all_ranks"], method
        assert o["trace"] == o["trace_single"], method


class _FakeComm:
    """The all-gather of a torch.distributed group whose ranks hold the given (n_offset, N, n_global) rows."""
    def __init__(self, rows):
        self.rows, self.world, self.rank = rows, len(rows), 0

    def allgather(self, t):
        return torch.tensor(self.rows, dtype=t.dtype, device=t.device)


@pytest.mark.parametrize("rows, ok", [
    ([(0, 5, 12), (5, 4, 12), (9, 3, 12)], True),
    ([(0, 12, 12), (0, 12, 12)], False),                      # every rank holds the whole task
    ([(0, 5, 12), (6, 6, 12)], False),                        # a gap
    ([(5, 7, 12), (0, 5, 12)], False),                        # ranges not in rank order
    ([(0, 5, 12), (5, 4, 12)], False),                        # short of the task
    ([(0, 6, 12), (6, 6, 13)], False),                        # ranks disagree on the task size
])
def test_one_process_per_gpu_requires_the_ranks_to_tile_the_task(rows, ok):
    from coda_b200.baselines import _check_rank_ranges
    off, n, ng = rows[0]
    preds = torch.zeros(2, n, 3)
    if ok:
        _check_rank_ranges(preds, off, n, ng, _FakeComm(rows))
    else:
        with pytest.raises(ValueError, match="N-range|cover"):
            _check_rank_ranges(preds, off, n, ng, _FakeComm(rows))


@pytest.mark.gpu
def test_sharding_arguments_are_rejected_under_one_process_per_gpu():
    from coda_b200 import IID, TensorDataset
    from coda_b200.synth import synth
    p, l = synth(4, 50, 3, 1)
    with pytest.raises(ValueError, match="torch.distributed"):
        IID(TensorDataset(p.cuda(), l.cuda()), None, shards=2, comm=_FakeComm([(0, 50, 50), (50, 50, 100)]))


def _dyadic_weights(g, labeled):
    """Small integer weights whose sum over the unlabeled items is a power of two P: every w / P is exact in fp32 and
    every running sum of them is exact in fp64, so a draw has one right answer whatever the summation order."""
    w = torch.randint(0, 4, labeled.shape, generator=g).double()
    unl = torch.nonzero(labeled == 0).flatten()
    if len(unl):
        s = int(w[unl].sum())
        p = 1 << max(0, (s - 1).bit_length())
        d = p - s
        w[unl] += d // len(unl)
        w[unl[torch.randperm(len(unl), generator=g)[:d % len(unl)]]] += 1
        assert int(w[unl].sum()) == p
    return w.float()


@pytest.mark.gpu
def test_exchange_entry_points_without_peers_match_a_host_evaluation():
    """Each selection entry point with x == NULL (world 1) against an evaluation on the host: the extreme and its ties,
    the k-th tie, the weighted total and the weighted draw.  With one shard no exchange waits, so no flag is set."""
    from coda_b200 import _native as nat
    lib = nat.load()
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(9)
    for N in (1, 37, 4096, 70_001):
        v = torch.randint(0, 6, (N,), generator=g).float()                # many exact ties
        labeled = (torch.rand(N, generator=g) < 0.3).to(torch.uint8)
        w = _dyadic_weights(g, labeled)
        unl = labeled == 0
        nb = int(lib.coda_b200_select_blocks(N))
        pi = torch.empty(2 * nb, dtype=torch.int64, device=dev)
        pf = torch.empty(2 * nb, dtype=torch.float64, device=dev)
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        s = torch.cuda.current_stream(dev).cuda_stream
        vd, wd, ld = v.to(dev), w.to(dev), labeled.to(dev)
        for want_max in (0, 1):
            bx = torch.full((4,), -7, dtype=torch.int64, device=dev)
            nat.call("coda_b200_select_extreme_xchg", vd.data_ptr(), ld.data_ptr(), N, want_max, pi.data_ptr(),
                     bx.data_ptr(), None, flags.data_ptr(), s)
            ties = torch.empty(0, dtype=torch.int64)
            bits, cnt = 0, 0
            if unl.any():
                best = v[unl].max() if want_max else v[unl].min()
                ties = torch.nonzero(unl & (v == best)).flatten()
                bits, cnt = int(np.float32(best.item()).view(np.uint32)), len(ties)
            assert bx.tolist() == [bits, cnt, 0, cnt], (N, want_max)
            for k in sorted({0, cnt // 2, max(0, cnt - 1)}):
                o = torch.full((1,), -7, dtype=torch.int64, device=dev)
                nat.call("coda_b200_select_kth_xchg", vd.data_ptr(), ld.data_ptr(), N, pi.data_ptr(), bx.data_ptr(), k, 0,
                         o.data_ptr(), None, flags.data_ptr(), s)
                assert o.tolist() == [int(ties[k]) if k < cnt else -1], (N, want_max, k)
        t = torch.empty(2, dtype=torch.float64, device=dev)
        nat.call("coda_b200_weighted_total_xchg", wd.data_ptr(), ld.data_ptr(), N, pf.data_ptr(), t.data_ptr(), None,
                 flags.data_ptr(), s)
        total = float(w[unl].double().sum())
        assert t.tolist() == [total, float(unl.sum())], N
        q = (w / np.float32(total)) if total else w                       # exact: total is a power of two
        items = torch.nonzero(unl).flatten()
        cum = torch.cumsum(q[items].double(), 0)
        for u in (0.0, 0.25, 0.5, 0.999999):
            o = torch.full((3,), -7, dtype=torch.int64, device=dev)
            nat.call("coda_b200_weighted_draw_xchg", wd.data_ptr(), ld.data_ptr(), N, t.data_ptr(), u, 0, pf.data_ptr(),
                     o.data_ptr(), None, flags.data_ptr(), s)
            if not len(items):
                want = [-1, -1, 0]
            else:
                past = torch.nonzero(cum > u * float(cum[-1])).flatten()       # bisect_right, the last item if none
                pos = int(past[0]) if len(past) else len(items) - 1
                i = int(items[pos])
                want = [pos, i, int(np.float32(q[i].item()).view(np.uint32))]
            assert o.tolist() == want, (N, u)
        src = torch.arange(13, dtype=torch.int16, device=dev)
        dst = torch.zeros(13, dtype=torch.int16, device=dev)
        nat.call("coda_b200_owner_share", src.data_ptr(), 26, 1, dst.data_ptr(), None, flags.data_ptr(), s)
        assert torch.equal(src, dst)
        assert int(flags.item()) == 0


@pytest.mark.gpu
def test_sharded_losses_of_another_dtype_are_shared_as_fp32():
    """A loss_fn returning float64 works on shards as on one shard (the shared losses are rounded to fp32)."""
    from coda.options import LOSS_FNS
    from coda_b200 import ActiveTesting, IID, TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(16, 3000, 7, 2)

    def loss64(p, l, **kw):
        return LOSS_FNS["acc"](p, l, **kw).double()
    for cls in (IID, ActiveTesting):
        runs = []
        for shards in (1, 2):
            _seed_all()
            sel = cls(TensorDataset(preds.cuda(), labels.cuda()), loss64, shards=shards)
            runs.append(_trace(sel, labels, 12))
            sel.close()
        if cls is IID:                                    # 0 / 1 losses: the same risk sums in either width
            assert runs[0] == runs[1]
        else:                                             # the LURE means are taken in fp32 instead of fp64
            assert [t[:2] for t in runs[0]] == [t[:2] for t in runs[1]]
