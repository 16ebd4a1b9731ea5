"""Parity of the CUDA path (through the C ABI / coda_b200.CODA) with the reference goldens and the CPU oracle.
Run on an H100:  python -m pytest tests -m gpu -x -q

Tolerances (SURVEY.md 8c; the reference is fp32 with a measured EIG noise floor of ~1.2e-6):
  EIG vector            abs 5e-6          P(best) / pi_hat      abs 1e-5 (north_star: 1e-4)
  pi_hat_xi             rel 5e-6          dirichlet update      one fp32 add: rel 2e-7 of the golden row
  selected index        identical wherever the reference's top-1/top-2 gap exceeds 1e-5, else epsilon-optimal
"""
import random

import numpy as np
import pytest
import torch

from helpers import coda_oracle, golden_names, golden_slab, load_golden

pytestmark = pytest.mark.gpu

EIG_ATOL = 5e-6


def _mk(preds, labels=None, **kw):
    from coda_b200 import CODA, TensorDataset
    dev = torch.device("cuda:0")
    return CODA(TensorDataset(preds.to(dev), None if labels is None else labels.to(dev)), **kw)


def _check_pick(ref_eig, idx, golden_idx):
    """epsilon-optimality protocol (SURVEY.md 8c-3)."""
    top = np.sort(ref_eig[~np.isnan(ref_eig)])[::-1]
    gap = top[0] - top[1] if len(top) > 1 else np.inf
    assert ref_eig[idx] >= top[0] - EIG_ATOL
    if gap > 1e-5:
        assert idx == golden_idx


@pytest.mark.parametrize("mode", ["incremental", "recompute", "recompute_all"])
@pytest.mark.parametrize("name", [n for n in golden_names() if "cfg2" not in n and "h256" not in n])
def test_golden_trajectory(name, mode):
    g = load_golden(name)
    preds, labels = golden_slab(g)
    random.seed(0)
    sel = _mk(preds, labels, mode=mode, **g["ctor"])
    eng = sel.engine
    # construction: hard predictions / unanimity are integer work -> exact
    ref_hard = preds.argmax(-1).T.numpy()
    assert np.array_equal(eng.hard.cpu().numpy().astype(np.int64) & 0xFFFF, ref_hard)
    assert np.array_equal(eng.disagree.cpu().numpy().astype(bool),
                          coda_oracle.disagreement_mask(preds.argmax(-1)).numpy())
    np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), g["init_dirichlets"], rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), g["init_pi_hat"], rtol=2e-6)
    np.testing.assert_allclose(sel.pi_hat_xi.cpu().numpy(), g["init_pi_hat_xi"], rtol=5e-6, atol=1e-9)
    b = sel.get_best_model_prediction()
    assert b.dim() == 0 and b.dtype == torch.int64 and int(b) == int(g["init_best_model"])     # trap T10
    pb = sel.get_pbest()
    assert tuple(pb.shape) == (1, int(g["H"]))
    np.testing.assert_allclose(pb.cpu().numpy(), g["init_pbest"], atol=1e-5)
    for k in range(int(g["steps"])):
        idx, q = sel.get_next_item_to_label()
        assert isinstance(idx, int) and isinstance(q, float)
        ref = g["eig"][k]
        cand = ~np.isnan(ref)
        assert sel.last_report["n_cand"] == int(g["n_cand"][k]) or not sel.last_report["use_a"]
        np.testing.assert_allclose(eng.eig.cpu().numpy()[cand], ref[cand], atol=EIG_ATOL)
        _check_pick(ref, idx, int(g["idx"][k]))
        assert abs(q - float(g["q"][k])) < EIG_ATOL or idx != int(g["idx"][k])
        gi = int(g["idx"][k])                     # teacher forcing: follow the reference's pick
        t = int(labels[gi])
        sel.add_label(gi, t, q)
        assert int(sel.get_best_model_prediction()) == int(g["best_model"][k])
        np.testing.assert_allclose(sel.get_pbest().cpu().numpy()[0], g["pbest"][k], atol=1e-5)
        np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), g["pi_hat"][k], rtol=2e-6)
        np.testing.assert_allclose(sel.dirichlets[:, t].cpu().numpy(), g["dir_row"][k], rtol=3e-7, atol=0)
        np.testing.assert_allclose(sel.pi_hat_xi[:64].cpu().numpy(), g["xi_head"][k], rtol=5e-6, atol=1e-9)
    np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), g["final_dirichlets"], rtol=2e-6, atol=1e-7)
    assert sel.step == int(g["steps"]) + 1
    assert sel.labeled_idxs == [int(i) for i in g["idx"]]
    assert len(sel.unlabeled_idxs) == int(g["N"]) - int(g["steps"])


def test_free_running_matches_reference_indices():
    """No teacher forcing: on this golden the reference's top-1 gaps are > 1e-5, so the picks must be identical."""
    g = load_golden("traj_small_h32_n3000_c10")
    preds, labels = golden_slab(g)
    random.seed(0)
    sel = _mk(preds, labels)
    picks = []
    for k in range(int(g["steps"])):
        idx, q = sel.get_next_item_to_label()
        picks.append(idx)
        sel.add_label(idx, int(labels[idx]), q)
        sel.get_best_model_prediction()
    assert picks == [int(i) for i in g["idx"]]
    np.testing.assert_allclose(sel.get_pbest().cpu().numpy()[0], g["pbest"][-1], atol=1e-5)
    assert sel.stochastic == bool(g["stochastic"])


def test_cfg2_golden_if_present():
    """BASELINE.json configs[1]: synthetic M=64 N=50k C=10 against the reference's own CPU trajectory."""
    names = [n for n in golden_names() if "cfg2" in n]
    if not names:
        pytest.skip("cfg2 golden not generated")
    g = load_golden(names[0])
    preds, labels = golden_slab(g)
    random.seed(0)
    sel = _mk(preds, labels)
    for k in range(int(g["steps"])):
        idx, q = sel.get_next_item_to_label()
        ref = g["eig"][k]
        cand = ~np.isnan(ref)
        np.testing.assert_allclose(sel.engine.eig.cpu().numpy()[cand], ref[cand], atol=EIG_ATOL)
        _check_pick(ref, idx, int(g["idx"][k]))
        gi = int(g["idx"][k])
        sel.add_label(gi, int(labels[gi]), q)
        assert int(sel.get_best_model_prediction()) == int(g["best_model"][k])
        np.testing.assert_allclose(sel.get_pbest().cpu().numpy()[0], g["pbest"][k], atol=1e-5)
        np.testing.assert_array_equal(sel.dirichlets[:, int(labels[gi])].cpu().numpy() > 0, True)
        np.testing.assert_allclose(sel.dirichlets[:, int(labels[gi])].cpu().numpy(), g["dir_row"][k], rtol=3e-7)


def test_oracle_on_fresh_seed_and_odd_shapes():
    """Not a golden: a shape no fixture covers (H not a multiple of 32, C not a multiple of 4), oracle run live."""
    from coda_b200.synth import synth
    preds, labels = synth(37, 700, 9, seed=11)
    random.seed(0)
    ora = coda_oracle.OracleSelector(preds)
    random.seed(0)
    sel = _mk(preds, labels)
    for _ in range(3):
        i_ref, q_ref = ora.get_next_item_to_label()
        i, q = sel.get_next_item_to_label()
        got = sel.engine.eig.cpu().numpy()[np.asarray(ora.last_cand)]
        np.testing.assert_allclose(got, ora.last_q.numpy(), atol=EIG_ATOL)
        assert i == i_ref
        ora.add_label(i, int(labels[i]), q_ref)
        sel.add_label(i, int(labels[i]), q)
        assert int(ora.get_best_model_prediction()) == int(sel.get_best_model_prediction())
        np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), ora.get_pbest().numpy(), atol=1e-5)


def test_edge_unanimous_fallback_and_h2():
    """Every model unanimous everywhere: the prefilter is empty and the candidate set falls back to all
    unlabeled items (coda.py:239); H=2 exercises the smallest leave-one-out product."""
    C, H, N = 4, 2, 40
    g = torch.Generator().manual_seed(3)
    y = torch.randint(0, C, (N,), generator=g)
    u = torch.rand((N, C), generator=g) * 0.05
    base = (u / u.sum(-1, keepdim=True) * 0.3)[None].repeat(H, 1, 1)
    base[:, torch.arange(N), y] += 0.7                       # both models predict y, item-specific scores
    random.seed(7)
    ora = coda_oracle.OracleSelector(base.clone())
    i_ref, q_ref = ora.get_next_item_to_label()
    sel = _mk(base, y)
    assert not bool(sel.engine.disagree.any())
    i, q = sel.get_next_item_to_label()
    assert not sel.last_report["use_a"] and sel.last_report["n_cand"] == 0
    np.testing.assert_allclose(sel.engine.eig.cpu().numpy(), ora.last_q.numpy(), atol=EIG_ATOL)
    assert ora.last_q.numpy()[i] >= ora.last_q.numpy().max() - EIG_ATOL and abs(q - q_ref) < EIG_ATOL


def test_exact_ties_consume_python_rng_like_the_reference():
    """coda.py:306-311: two items with identical predictions tie exactly; the pick is random.choice over the
    tied candidates in ascending order and `stochastic` flips.  Same RNG state => same pick as the oracle."""
    from coda_b200.synth import synth
    preds, labels = synth(10, 400, 6, seed=8)
    random.seed(1)
    first, _ = coda_oracle.OracleSelector(preds).get_next_item_to_label()
    twin = (first + 137) % 400
    preds[:, twin] = preds[:, first]
    for seed in (1, 2, 3, 4):
        random.seed(seed)
        ora = coda_oracle.OracleSelector(preds)
        i_ref, q_ref = ora.get_next_item_to_label()
        after_ref = random.getstate()
        assert ora.stochastic and i_ref in (first, twin)
        random.seed(seed)
        sel = _mk(preds, labels)
        i, q = sel.get_next_item_to_label()
        assert sel.last_report["n_ties"] == 2 and sel.stochastic
        assert i == i_ref and abs(q - q_ref) < EIG_ATOL and random.getstate() == after_ref


def test_modes_agree_and_incremental_is_exact():
    """Size-independent property: the cached-row path must reproduce a from-scratch recompute after many labels."""
    from coda_b200.synth import synth
    preds, labels = synth(48, 20000, 20, seed=5)
    sels = {}
    for mode in ("incremental", "recompute", "recompute_all"):
        random.seed(0)
        sels[mode] = _mk(preds, labels, mode=mode)
    for k in range(12):
        picks = {}
        for mode, s in sels.items():
            picks[mode] = s.get_next_item_to_label()
        e_inc = sels["incremental"].engine.eig.cpu().numpy()
        e_rec = sels["recompute"].engine.eig.cpu().numpy()
        e_all = sels["recompute_all"].engine.eig.cpu().numpy()
        np.testing.assert_allclose(e_inc, e_rec, atol=2e-8, rtol=0)     # same tables, same rows: summation order only
        np.testing.assert_allclose(e_inc, e_all, atol=1e-6, rtol=0)     # rank-1 vs full refresh of the marginals
        idx, q = picks["incremental"]
        for s in sels.values():
            s.add_label(idx, int(labels[idx]), q)
            s.get_best_model_prediction()
        np.testing.assert_allclose(sels["incremental"].get_pbest().cpu().numpy(),
                                   sels["recompute_all"].get_pbest().cpu().numpy(), atol=1e-6)
    # rank-1 marginal refresh (coda.py:319 restated) vs the full slab pass after 12 labels
    np.testing.assert_allclose(sels["incremental"].pi_hat_xi.cpu().numpy(),
                               sels["recompute_all"].pi_hat_xi.cpu().numpy(), rtol=2e-6, atol=1e-9)
    xi = sels["incremental"].pi_hat_xi
    np.testing.assert_allclose(xi.sum(-1).cpu().numpy(), 1.0, atol=1e-5)
    assert abs(float(sels["incremental"].pi_hat.sum()) - 1.0) < 1e-5


def test_row_structure_invariants():
    """Entry lists (item-major), heavy rows (contiguous per item, ascending class) and the class-major work list the
    row kernels tile over (zmask, row_of) describe exactly the hard predictions."""
    from coda_b200.synth import synth
    preds, labels = synth(40, 3000, 12, seed=2, dense=True)
    sel = _mk(preds, labels)
    e = sel.engine
    H, C, T = e.H, e.C, e.T
    hard = preds.argmax(-1).T.numpy()                                     # (N, H)
    ent_off = e.ent_off.cpu().numpy()
    heavy_off = e.heavy_off.cpu().numpy()
    ent_row = e.ent_row.cpu().numpy()
    ent_cls = e.ent_cls.cpu().numpy().astype(np.int64) & 0xFFFF
    zmask = e.zmask.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
    row_of = e.row_of.cpu().numpy()
    base = e.cls_base_host
    assert e.npairs == T + e.n_heavy == T + int(heavy_off[-1]) and len(row_of) == e.npairs
    assert sorted(row_of.tolist()) == list(range(e.npairs))               # the work list is a permutation of the rows
    pos_of_row = np.empty(e.npairs, dtype=np.int64)
    pos_of_row[row_of] = np.arange(e.npairs)

    def bits(q):
        return [h for h in range(H) if (zmask[q, h >> 5] >> (h & 31)) & 1]
    for c in range(C):                                                    # templates: class-major rows c*(1+H)+k
        for k in (0, 1, H // 2, H):
            q = base[c] + k
            assert row_of[q] == c * (1 + H) + k and bits(q) == ([] if k == 0 else [k - 1])
    for n in list(range(0, 3000, 97)) + [2999]:
        classes = sorted(set(hard[n].tolist()))
        seg = slice(ent_off[n], ent_off[n + 1])
        assert ent_cls[seg].tolist() == classes                           # one entry per distinct class, ascending
        rows = ent_row[seg]
        heavy_rows = rows[rows >= T]
        assert heavy_rows.tolist() == list(range(T + heavy_off[n], T + heavy_off[n + 1]))   # contiguous, in entry order
        for c, row in zip(classes, rows.tolist()):
            members = np.nonzero(hard[n] == c)[0]
            if len(members) == 1:
                assert row == c * (1 + H) + 1 + members[0]                # singleton template row
            else:
                q = pos_of_row[row]
                assert row >= T and base[c] + 1 + H <= q < base[c + 1] and bits(q) == members.tolist()


def test_fixed_point_sums_are_shard_invariant():
    """The sufficient statistics exchanged between GPUs (coda.py:42 sums, coda.py:232 sums) are int64 fixed point:
    accumulating two half-slabs gives bit-identical results to one pass (through the raw C ABI)."""
    from coda_b200 import _native as nat
    from coda_b200.synth import synth
    lib = nat.load()
    H, N, C = 16, 5000, 7
    preds, _ = synth(H, N, C, seed=9)
    dev = torch.device("cuda:0")
    P = preds.to(dev)
    st = torch.cuda.current_stream().cuda_stream

    def conf(p):
        n = p.shape[1]
        hard = torch.empty((n, H), dtype=torch.int16, device=dev)
        pseudo = torch.empty(n, dtype=torch.int32, device=dev)
        dis = torch.empty(n, dtype=torch.uint8, device=dev)
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        out = torch.zeros((H, C, C), dtype=torch.int64, device=dev)
        nat.check(lib.coda_b200_scan_slab(p.data_ptr(), n * C, H, n, C, hard.data_ptr(), pseudo.data_ptr(), dis.data_ptr(),
                                          None, flags.data_ptr(), st))
        nat.check(lib.coda_b200_confusion_accum(p.data_ptr(), n * C, pseudo.data_ptr(), H, n, C, 40, out.data_ptr(), st))
        return out, pseudo
    whole, pseudo = conf(P)
    a, _ = conf(P[:, :2300].contiguous())
    b, _ = conf(P[:, 2300:].contiguous())
    assert torch.equal(whole, a + b)
    # the class-sorted register variant produces the same bits as the shared-memory-atomics variant
    order = torch.argsort(pseudo).to(torch.int32)
    sorted_out = torch.zeros_like(whole)
    nat.check(lib.coda_b200_confusion_sorted(P.data_ptr(), N * C, pseudo.data_ptr(), order.data_ptr(), H, N, C, 40,
                                             sorted_out.data_ptr(), st))
    # an N-range VIEW of the slab (model stride = the full task's) gives the same sums as a contiguous copy of it
    view, _ = conf(P[:, :2300].contiguous())
    hard = torch.empty((2300, H), dtype=torch.int16, device=dev)
    ps2 = torch.empty(2300, dtype=torch.int32, device=dev)
    dis = torch.empty(2300, dtype=torch.uint8, device=dev)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    out = torch.zeros((H, C, C), dtype=torch.int64, device=dev)
    nat.check(lib.coda_b200_scan_slab(P.data_ptr(), N * C, H, 2300, C, hard.data_ptr(), ps2.data_ptr(), dis.data_ptr(),
                                      None, flags.data_ptr(), st))
    nat.check(lib.coda_b200_confusion_accum(P.data_ptr(), N * C, ps2.data_ptr(), H, 2300, C, 40, out.data_ptr(), st))
    assert torch.equal(out, view)
    assert torch.equal(whole, sorted_out)
    ref = torch.einsum("nc,hnj->hcj", torch.nn.functional.one_hot(pseudo.long().cpu(), C).float(), preds)
    np.testing.assert_allclose((whole.double() / 2 ** 40).cpu().numpy(), ref.numpy(), rtol=2e-6, atol=1e-6)


def test_api_and_error_behaviour():
    from coda_b200 import CODA, TensorDataset
    from coda_b200.synth import synth
    preds, labels = synth(8, 300, 5, seed=1)
    with pytest.raises(RuntimeError, match="no CPU path"):
        CODA(TensorDataset(preds, labels))                       # CPU tensor: refuse loudly, never fall back
    sel = _mk(preds, labels, q="bogus")
    with pytest.raises(NotImplementedError):                     # coda.py:297
        sel.get_next_item_to_label()
    sel = _mk(preds, labels)
    idx, q = sel.get_next_item_to_label()
    sel.add_label(idx, int(labels[idx]), q)
    with pytest.raises(ValueError):                              # coda.py:323 list.remove
        sel.add_label(idx, int(labels[idx]), q)
    sel.unlabeled_idxs.remove(5)                                 # demo/app.py:188: skip an item without labeling it
    for _ in range(3):
        i2, q2 = sel.get_next_item_to_label()
        assert i2 not in (idx, 5)
        sel.add_label(i2, int(labels[i2]), q2)
    assert len(sel.unlabeled_idxs) == 300 - 5 and 5 not in sel.unlabeled_idxs
    bad = preds.clone()
    bad[3, 17, 2] = float("nan")
    with pytest.raises(RuntimeError, match="NUMERIC ERROR"):     # util.py:20-25
        _mk(bad, labels)
    with pytest.raises(ValueError, match="post-softmax"):
        _mk(preds * 3.0, labels)

    class A:  # coda.py:205-213
        prefilter_n = 0; alpha = 0.9; learning_rate = 0.01; multiplier = 2.0; no_diag_prior = False; q = "eig"
    s2 = CODA.from_args(TensorDataset(preds.cuda(), labels.cuda()), A)
    assert s2.get_next_item_to_label()[0] == _mk(preds, labels).get_next_item_to_label()[0]


def test_prefilter_n_subsample_path():
    """coda.py:221-223 (--prefilter-n): same RNG consumption and pick as the oracle on the subsample."""
    from coda_b200.synth import synth
    preds, labels = synth(10, 600, 6, seed=8)
    random.seed(5)
    ora = coda_oracle.OracleSelector(preds, prefilter_n=50)
    i_ref, q_ref = ora.get_next_item_to_label()
    state_ref = random.getstate()
    random.seed(5)
    sel = _mk(preds, labels, prefilter_n=50)
    i, q = sel.get_next_item_to_label()
    assert i == i_ref and abs(q - q_ref) < EIG_ATOL and random.getstate() == state_ref and sel.stochastic


def test_tensor_core_rows_match_simt_rows(monkeypatch):
    """pairs_tc.cu (wgmma, bf16 limbs) against pairs.cu (fp32 SIMT) on the same tables: per-item EIG and P(best)."""
    from coda_b200.synth import synth
    for (H, N, C, seed) in [(256, 6000, 20, 3), (40, 3000, 12, 2), (100, 2000, 7, 6)]:
        preds, labels = synth(H, N, C, seed=seed)
        out = {}
        for tc in ("1", "0"):
            monkeypatch.setenv("CODA_B200_TC", tc)
            random.seed(0)
            s = _mk(preds, labels, mode="incremental")
            assert s.engine.use_tc == (tc == "1")
            eigs = []
            for k in range(3):
                idx, q = s.get_next_item_to_label()
                eigs.append(s.engine.eig.cpu().numpy().copy())
                if k == 0:
                    first = idx
                s.add_label(first + k, int(labels[first + k]), q)      # same labels on both paths
                s.get_best_model_prediction()
            out[tc] = (np.stack(eigs), s.get_pbest().cpu().numpy())
        np.testing.assert_allclose(out["1"][0], out["0"][0], atol=2e-7, rtol=0)
        np.testing.assert_allclose(out["1"][1], out["0"][1], atol=1e-7, rtol=0)


def test_wide_model_axis_uses_simt_rows_and_matches_oracle():
    """H = 300 (Hp = 320 > 256): beyond the tensor-core tile, the fp32 SIMT kernel with 10-word masks takes over."""
    from coda_b200.synth import synth
    preds, labels = synth(300, 260, 5, seed=13)
    random.seed(0)
    ora = coda_oracle.OracleSelector(preds)
    random.seed(0)
    sel = _mk(preds, labels)
    assert not sel.engine.use_tc and sel.engine.W == 10
    for _ in range(2):
        i_ref, q_ref = ora.get_next_item_to_label()
        i, q = sel.get_next_item_to_label()
        np.testing.assert_allclose(sel.engine.eig.cpu().numpy()[np.asarray(ora.last_cand)], ora.last_q.numpy(), atol=EIG_ATOL)
        assert ora.last_q.numpy()[ora.last_cand.index(i)] >= float(ora.last_q.max()) - EIG_ATOL
        ora.add_label(i_ref, int(labels[i_ref]), q_ref)
        sel.add_label(i_ref, int(labels[i_ref]), q)
        np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), ora.get_pbest().numpy(), atol=1e-5)


def test_degenerate_single_model_and_two_classes():
    """H = 1: P(best) is 1, every EIG is ~0, so every candidate ties (more than the device tie buffer holds):
    the pick is random.choice over ALL candidates exactly like the reference (coda.py:306-311).  C = 2 is the
    smallest class count the Dirichlet prior supports (coda.py:57 divides by C - 1)."""
    from coda_b200.synth import synth
    preds, labels = synth(1, 400, 2, seed=21)
    random.seed(9)
    ora = coda_oracle.OracleSelector(preds)
    i_ref, q_ref = ora.get_next_item_to_label()
    st_ref = random.getstate()
    random.seed(9)
    sel = _mk(preds, labels)
    i, q = sel.get_next_item_to_label()
    assert sel.last_report["n_ties"] == 400 and sel.stochastic and ora.stochastic
    assert abs(q - q_ref) < EIG_ATOL and abs(q) < EIG_ATOL
    if int(torch.isclose(ora.last_q, ora.last_q.max(), rtol=1e-8).sum()) == 400:
        assert i == i_ref and random.getstate() == st_ref
    np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), [[1.0]], atol=1e-6)
    sel.add_label(i, int(labels[i]), q)
    assert int(sel.get_best_model_prediction()) == 0


@pytest.mark.parametrize("q", ["iid", "uncertainty"])
def test_ablation_acquisitions_match_oracle(q):
    """coda.py:287-295: q='iid' / q='uncertainty' (paper ablation 2) with the reference's tie rule and RNG use."""
    from coda_b200.synth import synth
    preds, labels = synth(12, 500, 6, seed=17)
    random.seed(4)
    ora = coda_oracle.OracleSelector(preds, q=q)
    random.seed(4)
    sel = _mk(preds, labels, q=q)
    for _ in range(4):
        st = random.getstate()
        i_ref, q_ref = ora.get_next_item_to_label()
        after = random.getstate()
        random.setstate(st)
        i, qq = sel.get_next_item_to_label()
        assert i == i_ref and abs(qq - q_ref) < 1e-6 and random.getstate() == after
        ora.add_label(i, int(labels[i]), q_ref)
        sel.add_label(i, int(labels[i]), qq)
        assert int(ora.get_best_model_prediction()) == int(sel.get_best_model_prediction())
    assert sel.stochastic == ora.stochastic


def test_main_py_loop_through_the_coda_shim(tmp_path):
    """The reference driver's loop (main.py:55-105: seed_all, true_losses, regret bookkeeping, the four calls per
    step) written against the `coda` shim exactly as main.py imports it, on a CUDA dataset loaded from disk;
    the regret trajectory must equal the one the CPU oracle produces."""
    import argparse
    from coda import CODA
    from coda.datasets import Dataset
    from coda.options import LOSS_FNS
    from coda.oracle import Oracle
    from coda_b200.synth import synth
    preds, labels = synth(16, 1500, 8, seed=23)
    torch.save(preds, str(tmp_path / "toy.pt"))
    torch.save(labels, str(tmp_path / "toy_labels.pt"))
    args = argparse.Namespace(prefilter_n=0, alpha=0.9, learning_rate=0.01, multiplier=2.0, no_diag_prior=False, q="eig",
                              iters=6)
    dataset = Dataset(str(tmp_path / "toy.pt"), device=torch.device("cuda:0"))          # main.py:114
    oracle = Oracle(dataset, loss_fn=LOSS_FNS["acc"])                                   # main.py:117-118
    random.seed(0); np.random.seed(0); torch.manual_seed(0)                             # main.py:19-26
    true_losses = oracle.true_losses(dataset.preds)                                     # main.py:57
    best_loss = min(true_losses)
    selector = CODA.from_args(dataset, args)                                            # main.py:67
    regrets = [float(true_losses[selector.get_best_model_prediction()] - best_loss)]   # main.py:83-84
    for _ in range(args.iters):                                                         # main.py:89-103
        chosen_idx, selection_prob = selector.get_next_item_to_label()
        true_class = oracle(chosen_idx)
        selector.add_label(chosen_idx, true_class, selection_prob)
        regrets.append(float(true_losses[selector.get_best_model_prediction()] - best_loss))
    # the same loop on the CPU oracle
    random.seed(0)
    ora = coda_oracle.OracleSelector(preds)
    tl = (1 - (preds.argmax(-1) == labels[None]).float()).mean(1)
    ref = [float(tl[ora.get_best_model_prediction()] - tl.min())]
    for _ in range(args.iters):
        i, q = ora.get_next_item_to_label()
        ora.add_label(i, int(labels[i]), q)
        ref.append(float(tl[ora.get_best_model_prediction()] - tl.min()))
    np.testing.assert_allclose(regrets, ref, atol=1e-6)
    assert selector.labeled_idxs == ora.labeled_idxs and selector.stochastic == ora.stochastic


@pytest.mark.parametrize("name", ["traj_small_h32_n3000_c10", "traj_nodiag_h10_n400_c6"])
def test_posterior_update_is_bit_exact_given_the_reference_state(name):
    """BASELINE configs[1] 'bit-match posterior': the construction sums differ from the reference's in summation order
    (so D agrees to ~1e-7), but the Bayesian update itself (coda.py:316-317) is one fp32 add per model.  Seeded with the
    reference's own initial dirichlets, every updated row must carry exactly the reference's bits, step after step."""
    g = load_golden(name)
    preds, labels = golden_slab(g)
    sel = _mk(preds, labels, **g["ctor"])
    sel.engine.D.copy_(torch.from_numpy(g["init_dirichlets"]).to(sel.engine.D.device))
    for k in range(int(g["steps"])):
        gi = int(g["idx"][k])
        t = int(labels[gi])
        sel.add_label(gi, t, 0.0)
        assert np.array_equal(sel.dirichlets[:, t].cpu().numpy(), g["dir_row"][k]), k
    assert np.array_equal(sel.dirichlets.cpu().numpy(), g["final_dirichlets"])


@pytest.mark.parametrize("C", [150, 300])
def test_many_classes_take_the_generic_kernels(C):
    """C > 128 leaves the register-resident fast paths (slab scan, confusion sums, rank-1 row pass, EIG assembly)
    for their generic twins; C = 300 also overflows the shared-memory confusion table."""
    from coda_b200.synth import synth
    preds, labels = synth(6, 220, C, seed=31)
    random.seed(0)
    ora = coda_oracle.OracleSelector(preds)
    random.seed(0)
    sel = _mk(preds, labels)
    np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), ora.dirichlets.numpy(), rtol=3e-6, atol=1e-7)
    for _ in range(2):
        i_ref, q_ref = ora.get_next_item_to_label()
        i, q = sel.get_next_item_to_label()
        np.testing.assert_allclose(sel.engine.eig.cpu().numpy()[np.asarray(ora.last_cand)], ora.last_q.numpy(), atol=EIG_ATOL)
        assert float(ora.last_q[ora.last_cand.index(i)]) >= float(ora.last_q.max()) - EIG_ATOL
        ora.add_label(i_ref, int(labels[i_ref]), q_ref)
        sel.add_label(i_ref, int(labels[i_ref]), q)
        np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), ora.get_pbest().numpy(), atol=1e-5)
        np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), ora.pi_hat.numpy(), rtol=5e-6, atol=1e-9)


@pytest.mark.parametrize("mode", ["incremental", "recompute"])
@pytest.mark.parametrize("name", golden_names())
def test_device_loop_follows_the_reference_trajectory(name, mode):
    """The host-free loop that produces bench.py's `value` (Engine.device_step: score -> merged arg-max -> label
    looked up on the device -> posterior update) against the reference's own free-running trajectory.  None of the
    goldens has an isclose tie (n_ties == 1 everywhere), so arg-max-first-index IS the reference's rule
    (coda.py:306-313) on these runs and every pick must be the reference's pick."""
    g = load_golden(name)
    if mode != "incremental" and int(g["N"]) > 20000:
        pytest.skip("large golden: product mode only")
    if int(g["n_ties"].max()) > 1:
        pytest.skip("the reference broke an isclose tie with random.choice on this golden (covered by the API-path tests)")
    preds, labels = golden_slab(g)
    sel = _mk(preds, labels, mode=mode, **g["ctor"])
    eng = sel.engine
    H, K = int(g["H"]), int(g["steps"])
    labels_dev = labels.to(eng.dev)
    hist_idx = torch.zeros(K, dtype=torch.int64, device=eng.dev)
    hist_q = torch.zeros(K, dtype=torch.float32, device=eng.dev)
    for k in range(K):
        eng.device_step(labels_dev, k, hist_idx, hist_q)
        gi = int(g["idx"][k])
        t = int(labels[gi])
        assert int(hist_idx[k]) == gi, (k, hist_idx.tolist(), g["idx"].tolist())
        assert abs(float(hist_q[k]) - float(g["q"][k])) < EIG_ATOL
        np.testing.assert_allclose(eng.m0[:H].cpu().numpy(), g["pbest"][k], atol=1e-5)
        np.testing.assert_allclose(eng.pi_hat.cpu().numpy(), g["pi_hat"][k], rtol=2e-6)
        np.testing.assert_allclose(eng.D[:, t].cpu().numpy(), g["dir_row"][k], rtol=3e-7, atol=0)
        assert int(eng.best_model[0]) == int(g["best_model"][k])
    if "final_dirichlets" in g:
        np.testing.assert_allclose(eng.D.cpu().numpy(), g["final_dirichlets"], rtol=2e-6, atol=1e-7)
    assert int(eng.labeled.sum()) == K
    eng.check_flags(sync=True)


def test_full_width_tensor_core_tile_against_the_reference():
    """H = 256, C = 100 (Hp = 256: 8 K-chunks, two column passes of k_pair_rows_tc) pinned to the reference's
    compute_pbest_beta_batched (coda.py:77-119) through a golden generated by the reference itself -- not to the
    SIMT twin.  Teacher-forced; EIG vector, pick, P(best), posterior rows."""
    names = [n for n in golden_names() if "h256" in n]
    if not names:
        pytest.skip("h256 golden not generated")
    g = load_golden(names[0])
    preds, labels = golden_slab(g)
    random.seed(0)
    sel = _mk(preds, labels)
    assert sel.engine.use_tc and sel.engine.Hp == 256
    np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), g["init_pbest"], atol=1e-5)
    for k in range(int(g["steps"])):
        idx, q = sel.get_next_item_to_label()
        ref = g["eig"][k]
        cand = ~np.isnan(ref)
        np.testing.assert_allclose(sel.engine.eig.cpu().numpy()[cand], ref[cand], atol=EIG_ATOL)
        _check_pick(ref, idx, int(g["idx"][k]))
        gi = int(g["idx"][k])
        sel.add_label(gi, int(labels[gi]), q)
        assert int(sel.get_best_model_prediction()) == int(g["best_model"][k])
        np.testing.assert_allclose(sel.get_pbest().cpu().numpy()[0], g["pbest"][k], atol=1e-5)
        np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), g["pi_hat"][k], rtol=5e-6)    # 256-model fp32 sums: order noise
        t = int(labels[gi])
        np.testing.assert_allclose(sel.dirichlets[:, t].cpu().numpy(), g["dir_row"][k], rtol=3e-7, atol=0)


def test_back_to_back_add_label_replays_a_label_history():
    """API-legal: several add_label calls with no get_next_item_to_label in between (replaying a label history).
    Every call must apply ITS OWN (idx, class) -- the pinned staging of the record must not be overwritten while an
    earlier copy is still queued behind the step kernels.  Checked against the oracle (small) and against a twin that
    synchronises between calls (large shard, where the kernels of one label take hundreds of microseconds)."""
    from coda_b200.synth import synth
    preds, labels = synth(10, 400, 6, seed=8)
    random.seed(0)
    ora = coda_oracle.OracleSelector(preds)
    sel = _mk(preds, labels)
    hist = [17, 230, 5, 399, 64, 128]
    for i in hist:
        ora.add_label(i, int(labels[i]), 0.0)
    for i in hist:
        sel.add_label(i, int(labels[i]), 0.0)                 # no sync, no fetch in between
    np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), ora.dirichlets.numpy(), rtol=3e-6, atol=1e-7)
    np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), ora.pi_hat.numpy(), rtol=5e-6)
    assert sorted(np.nonzero(sel.engine.labeled.cpu().numpy())[0].tolist()) == sorted(hist)
    np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), ora.get_pbest().numpy(), atol=1e-5)
    preds, labels = synth(64, 300000, 16, seed=6)
    a, b = _mk(preds, labels), _mk(preds, labels)
    hist = [7, 150001, 299999, 31337, 8, 123456, 222222, 9]
    for i in hist:
        a.add_label(i, int(labels[i]), 0.0)
    for i in hist:
        b.add_label(i, int(labels[i]), 0.0)
        torch.cuda.synchronize()
    assert torch.equal(a.dirichlets, b.dirichlets) and torch.equal(a.pi_hat, b.pi_hat)
    assert torch.equal(a.engine.labeled, b.engine.labeled) and torch.equal(a.get_pbest(), b.get_pbest())
    ia, ib = a.get_next_item_to_label(), b.get_next_item_to_label()
    assert ia == ib


def test_best_model_prediction_is_a_fresh_tensor():
    """coda.py:346 returns torch.argmax(...): a new tensor every call.  A caller keeping the result of an earlier
    step must not see it change when later steps run."""
    g = load_golden("traj_small_h32_n3000_c10")
    preds, labels = golden_slab(g)
    sel = _mk(preds, labels)
    kept = []
    for k in range(int(g["steps"])):
        gi = int(g["idx"][k])
        sel.add_label(gi, int(labels[gi]), 0.0)
        kept.append(sel.get_best_model_prediction())
    assert [int(b) for b in kept] == [int(x) for x in g["best_model"]]
    assert len({b.data_ptr() for b in kept}) == len(kept)


@pytest.mark.parametrize("shape", [(64, 20000, 20, 5), (37, 3001, 7, 11), (256, 6000, 100, 3), (12, 333, 33, 4)])
def test_marginal_refresh_variants_carry_identical_bits(shape, monkeypatch):
    """The two term paths of the rank-1 marginal refresh (the gather list in a constant-bank slot -- the default --, or
    in shared memory, which a selector gets once its device's slots are used up; CODA_B200_R1_CONST=0 at construction)
    do the same arithmetic in the same order: U, the fixed-point column sums and pi_hat carry identical bits after every
    label, for item counts / class counts that are not multiples of the tile or of four, with and without shadow slots."""
    import gc
    from coda_b200.synth import synth
    H, N, C, seed = shape
    preds, labels = synth(H, N, C, seed=seed)
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    for shadow_models in (None, "3"):
        if shadow_models:
            monkeypatch.setenv("CODA_B200_SHADOW_MODELS", shadow_models)
        else:
            monkeypatch.delenv("CODA_B200_SHADOW_MODELS", raising=False)
        gc.collect()                                          # selectors of earlier tests give their slots back
        monkeypatch.delenv("CODA_B200_R1_CONST", raising=False)
        sels = {"const": _mk(preds, labels)}
        monkeypatch.setenv("CODA_B200_R1_CONST", "0")
        sels["smem"] = _mk(preds, labels)
        monkeypatch.delenv("CODA_B200_R1_CONST")
        assert sels["const"].engine.const_slot >= 0 and sels["smem"].engine.const_slot == -1
        for k, i in enumerate([3, N // 2, N - 1, 17, N // 3]):
            for s in sels.values():
                s.add_label(i, int(labels[i]), 0.0)
                torch.cuda.synchronize()
            assert torch.equal(sels["const"].engine.U, sels["smem"].engine.U), (shape, shadow_models, k)
            assert torch.equal(sels["const"].engine.pisum, sels["smem"].engine.pisum)
            assert torch.equal(sels["const"].pi_hat, sels["smem"].pi_hat)
        picks = {v: s.get_next_item_to_label() for v, s in sels.items()}
        assert picks["const"] == picks["smem"]
        for s in sels.values():
            s.close()


@pytest.mark.parametrize("shape", [(256, 1000, 100, 1.0), (5, 128, 16, 1.0), (9, 700, 128, 1.0), (30, 257, 20, 3e5),
                                   (64, 4100, 52, 1e-3), (3, 40, 24, 1.0), (1, 300, 128, 1.0), (48, 100, 16, 1.0)])
def test_tensor_core_marginals_match_fp64(shape):
    """coda.py:227-229 on wgmma (k_pi_full_tc: two fp16 limbs per operand, accumulators folded every 4 models)
    against an fp64 contraction and against the fp32 SIMT kernel, through the raw C ABI: ragged last tile, class counts
    that are not a multiple of 16, a model count that is not a multiple of the drain group, Dirichlet parameters far
    outside the fp16 range (rescaled by a power of two inside), a slab VIEW (model stride larger than the shard), and
    bit-identical rows wherever the tile boundaries fall (the shard-count invariance)."""
    from coda_b200 import _native as nat
    lib = nat.load()
    H, N, C, dscale = shape
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(H * 1000 + C)
    preds = torch.softmax(3 * torch.randn((H, N + 40, C), generator=g), dim=-1).to(dev)
    D = (0.2 + 2 * torch.rand((H, C, C), generator=g)).to(dev)
    D += 5 * torch.eye(C, device=dev)
    D *= dscale
    st = torch.cuda.current_stream().cuda_stream
    ld = (N + 40) * C
    assert lib.coda_b200_pi_full_tc_ok(H, N, C, ld)
    scratch = torch.empty(int(lib.coda_b200_pi_full_tc_scratch_bytes(H, C)), dtype=torch.uint8, device=dev)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)

    def tc(first, n):
        U = torch.full((n, C), float("nan"), device=dev)
        view = preds[:, first:]
        nat.check(lib.coda_b200_pi_full_tc(view.data_ptr(), ld, D.data_ptr(), H, n, C, U.data_ptr(), scratch.data_ptr(),
                                           flags.data_ptr(), st), "pi_full_tc")
        torch.cuda.synchronize()
        return U
    U = tc(0, N)
    assert int(flags.item()) == 0
    ref = torch.einsum("hns,hcs->nc", preds[:, :N].double(), D.double())
    rel = ((U.double() - ref).abs() / ref).max().item()
    assert rel < 5e-6, rel                                     # the fp32 inputs are carried exactly; what is left is the
    xi, xr = U.double() / U.double().sum(1, keepdim=True), ref / ref.sum(1, keepdim=True)   # truncating accumulate of 4 models
    assert ((xi - xr).abs() / xr).max().item() < 2e-6          # (a common factor: it cancels in the row normalisation)
    simt = torch.empty((N, C), device=dev)
    nat.check(lib.coda_b200_pi_full(preds.data_ptr(), ld, D.data_ptr(), H, N, C, simt.data_ptr(), st), "pi_full")
    torch.cuda.synchronize()
    np.testing.assert_allclose(U.cpu().numpy(), simt.cpu().numpy(), rtol=1e-4)       # the fp32 FMA chain is the looser one
    rel_s = ((simt.double() - ref).abs() / ref).max().item()                          # an H*C-term FMA chain of non-negative
    print(f"[marginal] pi_full   SIMT H={H} N={N} C={C} (rel)   worst {rel_s:.3e}   bound {H * C * 2.0 ** -24:.1e}")
    assert rel_s <= H * C * 2.0 ** -24                                                 # terms: H*C u relative
    if H * C >= 20000:                                                                 # (H*C sequential roundings per entry)
        xs = simt.double() / simt.double().sum(1, keepdim=True)
        assert ((xi - xr).abs() / xr).max().item() < ((xs - xr).abs() / xr).max().item()
    # a shard that starts 40 items (not a tile multiple) later computes the same bits for the items both hold
    if N > 40 and (40 * C) % 4 == 0:
        V = tc(40, N)
        assert torch.equal(V[: N - 40], U[40:])
