"""fp16 / bf16 prediction slabs are read at their stored width and give bit-identical results to the fp32 path run on
their exact fp32 widening: per kernel through the raw C ABI, and end to end through CODA and the baselines."""
import hashlib
import pickle
import random

import numpy as np
import pytest
import torch

from coda_b200 import _native as nat
from coda_b200.synth import synth

DTYPES = [torch.float16, torch.bfloat16]
FMT = {torch.float32: nat.SLAB_F32, torch.float16: nat.SLAB_F16, torch.bfloat16: nat.SLAB_BF16}


def _p(t):
    return t.data_ptr() if t is not None else None


def _pair(H, N, C, dt, seed=0, off=0):
    """(16-bit slab, its fp32 widening), both N-range views at item offset ``off`` of a larger contiguous slab."""
    x, _ = synth(H, N + off + 3, C, seed=seed, dtype=dt)
    x = x.cuda()
    w = x.float()
    return x[:, off:off + N], w[:, off:off + N]


def _stride(t):
    return int(t.stride(0)) if t.shape[0] > 1 else t.shape[1] * t.shape[2]


def _scan(lib, x, ens=True):
    H, N, C = x.shape
    hard = torch.empty((N, H), dtype=torch.int16, device="cuda")
    pseudo = torch.empty(N, dtype=torch.int32, device="cuda")
    dis = torch.empty(N, dtype=torch.uint8, device="cuda")
    e = torch.empty((N, C), dtype=torch.float32, device="cuda") if ens else None
    flags = torch.zeros(1, dtype=torch.int32, device="cuda")
    nat.check(lib.coda_b200_scan_slab_x(_p(x), FMT[x.dtype], _stride(x), H, N, C, _p(hard), _p(pseudo), _p(dis), _p(e),
                                        _p(flags), None), "scan")
    torch.cuda.synchronize()
    return hard, pseudo, dis, e, flags


SHAPES = [(1, 1001, 5), (33, 1507, 10), (33, 1003, 12), (33, 777, 16), (24, 901, 100), (8, 513, 128), (5, 400, 130)]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("off", [0, 3])
def test_slab_kernels_match_fp32_widening(dt, shape, off):
    """scan (hard, pseudo, unanimity, E, flags), confusion sums (sorted and accumulating), the SIMT and tensor-core
    marginal passes and the shadow copy: 16-bit slab == fp32 widening, bit for bit."""
    lib = nat.load()
    H, N, C = shape
    x, w = _pair(H, N, C, dt, seed=H + C, off=off)
    a, b = _scan(lib, x), _scan(lib, w)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    pseudo = a[1]
    fx = 30
    for name in ("sorted", "accum"):
        if name == "sorted" and C > 128:
            continue
        outs = []
        for t in (x, w):
            conf = torch.zeros((H, C, C), dtype=torch.int64, device="cuda")
            if name == "sorted":
                order = torch.argsort(pseudo).to(torch.int32)
                rc = lib.coda_b200_confusion_sorted_x(_p(t), FMT[t.dtype], _stride(t), _p(pseudo), _p(order), H, N, C, fx,
                                                      _p(conf), None)
            else:
                rc = lib.coda_b200_confusion_accum_x(_p(t), FMT[t.dtype], _stride(t), _p(pseudo), H, N, C, fx, _p(conf), None)
            nat.check(rc, name)
            outs.append(conf)
        assert torch.equal(outs[0], outs[1]), name
    D = torch.rand((H, C, C), device="cuda") * 3 + 0.1
    for tc in (False, True):
        if tc and not lib.coda_b200_pi_full_tc_ok(H, N, C, N * C):
            assert not (C >= 16 and C <= 128 and C % 4 == 0)
            continue
        assert not tc or lib.coda_b200_pi_full_tc_ok_x(FMT[dt], H, N, C, _stride(x))
        outs = []
        for t in (x, w):
            U = torch.empty((N * C + 4,), dtype=torch.float32, device="cuda")
            flags = torch.zeros(1, dtype=torch.int32, device="cuda")
            if tc:
                scr = torch.empty((int(lib.coda_b200_pi_full_tc_scratch_bytes(H, C)),), dtype=torch.uint8, device="cuda")
                rc = lib.coda_b200_pi_full_tc_x(_p(t), FMT[t.dtype], _stride(t), _p(D), H, N, C, _p(U), _p(scr),
                                                _p(flags), None)
            else:
                rc = lib.coda_b200_pi_full_x(_p(t), FMT[t.dtype], _stride(t), _p(D), H, N, C, _p(U), None)
            nat.check(rc, "pi_full")
            torch.cuda.synchronize()
            assert int(flags.item()) == 0
            outs.append(U[: N * C])
        assert torch.equal(outs[0], outs[1]), ("tc" if tc else "simt")
    S = min(H, 3)
    order = torch.arange(H - 1, H - 1 - S, -1, dtype=torch.int32, device="cuda")
    cs = (N + 7) // 8 * 8
    sh = []
    for t in (x, w):
        T = torch.zeros((S, C, cs), dtype=t.dtype, device="cuda")
        nat.check(lib.coda_b200_shadow_build_x(_p(t), FMT[t.dtype], _stride(t), H, N, C, _p(order), S, cs, _p(T), None),
                  "shadow")
        sh.append(T)
    assert torch.equal(sh[0].float(), sh[1])


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_scan_flags_nan_and_range(dt):
    lib = nat.load()
    for bad, want in ((float("nan"), nat.FLAG_NONFINITE_INPUT), (1.5, nat.FLAG_RANGE_INPUT), (-0.25, nat.FLAG_RANGE_INPUT)):
        for C in (10, 100):
            x, w = _pair(4, 300, C, dt, seed=C)
            x = x.clone()
            x[2, 17, 3] = bad
            w = x.float()
            a, b = _scan(lib, x), _scan(lib, w)
            assert int(a[4].item()) & want
            for u, v in zip(a, b):
                assert torch.equal(u, v) or (u.is_floating_point() and torch.equal(u.isnan(), v.isnan()))


def _digest():
    return hashlib.sha256(pickle.dumps((random.getstate(), torch.get_rng_state().numpy().tobytes(),
                                        torch.cuda.get_rng_state().numpy().tobytes()))).hexdigest()


def _trace(sel, labels, steps):
    out = {"picks": [], "q": [], "eig": []}
    for _ in range(steps):
        idx, q = sel.get_next_item_to_label()
        if sel.q == "eig":
            out["eig"].append(sel.eig.cpu())
        out["picks"].append(int(idx))
        out["q"].append(float(q))
        sel.add_label(idx, int(labels[idx]), q)
    out["D"] = sel.dirichlets.cpu()
    out["pi_hat"] = sel.pi_hat.cpu()
    out["xi"] = sel.pi_hat_xi.cpu()
    out["pbest"] = sel.get_pbest().cpu()
    out["best"] = int(sel.get_best_model_prediction())
    out["stochastic"] = sel.stochastic
    out["rng"] = _digest()
    out["flags"] = [int(e.flags.item()) for e in sel.engines]
    return out


def _same(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if k == "eig":
            assert len(a[k]) == len(b[k])
            for u, v in zip(a[k], b[k]):
                assert torch.equal(u, v), k
        elif isinstance(a[k], torch.Tensor):
            assert torch.equal(a[k], b[k]), k
        else:
            assert a[k] == b[k], k


def _both(x, labels, steps=8, **kw):
    """Run CODA on the 16-bit slab and on its widening with the same seeds -> the two traces."""
    from coda_b200 import CODA, TensorDataset
    outs = []
    for t in (x, x.float()):
        random.seed(1)
        torch.manual_seed(1)
        sel = CODA(TensorDataset(t, labels), **kw)
        outs.append(_trace(sel, labels.cpu(), steps))
        sel.close()
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("shape", [(33, 1507, 12), (24, 901, 100), (16, 777, 16), (5, 400, 130)])
@pytest.mark.parametrize("shards", [1, 2, 3])
def test_coda_identical_on_16bit_slab(dt, shape, shards, monkeypatch):
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    H, N, C = shape
    x, labels = synth(H, N, C, seed=7, dtype=dt)
    a, b = _both(x.cuda(), labels.cuda(), shards=shards)
    _same(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("env", [{"CODA_B200_R1_CONST": "0"}, {"CODA_B200_SHADOW": "0"},
                                 {"CODA_B200_SHADOW_MODELS": "3"}, {"CODA_B200_TC": "0"}, {"CODA_B200_ENS": "0"},
                                 {"CODA_B200_PI_FULL": "simt"}])
def test_coda_identical_across_kernel_paths(dt, env, monkeypatch):
    """Each rank-1 refresh term path (constant bank / shared memory), the shadow off, capped and full."""
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    for shape in ((40, 1203, 100), (37, 1001, 10)):
        x, labels = synth(*shape, seed=3, dtype=dt)
        a, b = _both(x.cuda(), labels.cuda(), steps=10)
        _same(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("kw", [dict(mode="recompute"), dict(mode="recompute_all"), dict(q="iid"),
                                dict(q="uncertainty"), dict(prefilter_n=200)])
def test_coda_identical_modes_and_ablations(dt, kw, monkeypatch):
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    x, labels = synth(24, 901, 100, seed=5, dtype=dt)
    a, b = _both(x.cuda(), labels.cuda(), steps=6, **kw)
    _same(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_run_steps_graph_loop_identical(dt):
    from coda_b200 import CODA, TensorDataset
    x, labels = synth(32, 3000, 100, seed=2, dtype=dt)
    x, labels = x.cuda(), labels.cuda()
    outs = []
    for t in (x, x.float()):
        sel = CODA(TensorDataset(t, labels), shards=2)
        sel.run_steps(25, labels)
        h = sel.history()
        outs.append((h, sel.eig.cpu(), sel.get_pbest().cpu(), sel.pi_hat_xi.cpu()))
        sel.close()
    (h0, e0, p0, x0), (h1, e1, p1, x1) = outs
    for u, v in zip(h0, h1):
        assert np.array_equal(np.asarray(u), np.asarray(v))
    assert torch.equal(e0, e1) and torch.equal(p0, p1) and torch.equal(x0, x1)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_state_dict_resumes_across_slab_widths(dt, monkeypatch):
    """Saved on the fp32 widening, resumed on the 16-bit slab (and the reverse): the continuation is bit-exact."""
    from coda_b200 import CODA, TensorDataset
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    x, labels = synth(24, 901, 100, seed=9, dtype=dt)
    x, labels = x.cuda(), labels.cuda()
    lab = labels.cpu()
    for src, dst in ((x.float(), x), (x, x.float())):
        random.seed(4)
        torch.manual_seed(4)
        s0 = CODA(TensorDataset(src, labels))
        _trace(s0, lab, 5)
        sd = s0.state_dict()
        ref = _trace(s0, lab, 5)
        s0.close()
        s1 = CODA(TensorDataset(dst, labels))
        s1.load_state_dict(sd)
        got = _trace(s1, lab, 5)
        s1.close()
        _same(ref, got)


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("method", ["iid", "uncertainty", "activetesting", "vma", "model_picker"])
def test_baselines_identical_on_16bit_slab(dt, method):
    from coda.options import LOSS_FNS
    from coda_b200 import IID, VMA, ActiveTesting, ModelPicker, TensorDataset, Uncertainty
    cls = {"iid": IID, "uncertainty": Uncertainty, "activetesting": ActiveTesting, "vma": VMA}
    x, labels = synth(24, 600, 100, seed=11, dtype=dt)
    x, labels = x.cuda(), labels.cuda()
    outs = []
    for t in (x, x.float()):
        random.seed(3)
        torch.manual_seed(3)
        torch.cuda.manual_seed(3)
        ds = TensorDataset(t, labels)
        sel = ModelPicker(ds) if method == "model_picker" else cls[method](ds, LOSS_FNS["acc"])
        picks, qs, best = [], [], []
        for _ in range(12):
            idx, q = sel.get_next_item_to_label()
            picks.append(int(idx))
            qs.append(float(q))
            sel.add_label(idx, int(labels[idx]), q)
            best.append(int(sel.get_best_model_prediction()))
        risk = sel.get_risk_estimates().cpu() if hasattr(sel, "get_risk_estimates") else None
        outs.append((picks, qs, best, risk, _digest()))
    a, b = outs
    assert a[:3] == b[:3] and a[4] == b[4]
    assert (a[3] is None and b[3] is None) or torch.equal(a[3], b[3])


@pytest.mark.gpu
def test_keep_dtype_driver_logs_same_regrets(tmp_path, monkeypatch):
    """The coda shim's Dataset with CODA_B200_KEEP_DTYPE=1 keeps an fp16 file at its width; a CODA run on it logs the
    same picks and best models as the default fp32 load."""
    import coda.datasets
    from coda_b200 import CODA
    x, labels = synth(16, 700, 10, seed=1, dtype=torch.float16)
    f = str(tmp_path / "task.pt")
    torch.save(x, f)
    torch.save(labels, str(tmp_path / "task_labels.pt"))
    monkeypatch.setenv("CODA_B200_GRAPH", "0")
    outs = []
    for keep in ("1", "0"):
        monkeypatch.setenv("CODA_B200_KEEP_DTYPE", keep)
        ds = coda.datasets.Dataset(f, "cuda")
        assert ds.preds.dtype == (torch.float16 if keep == "1" else torch.float32)
        random.seed(0)
        sel = CODA(ds)
        regrets = []
        acc = (ds.preds.float().argmax(-1).cpu() == labels[None]).float().mean(1)
        for _ in range(10):
            idx, q = sel.get_next_item_to_label()
            sel.add_label(idx, int(ds.labels[idx]), q)
            regrets.append(float(acc.max() - acc[int(sel.get_best_model_prediction())]))
        outs.append(regrets)
        sel.close()
    assert outs[0] == outs[1]


@pytest.mark.gpu
@pytest.mark.parametrize("dt", DTYPES)
def test_eager_profile_names_16bit_entry_points_like_fp32(dt):
    """A profile restricted to an fp32 entry point's name also times its 16-bit twin, under that name."""
    from coda_b200 import CODA, TensorDataset
    x, labels = synth(16, 900, 20, seed=4, dtype=dt)
    x, labels = x.cuda(), labels.cuda()
    sel = CODA(TensorDataset(x, labels))
    eng = sel.engine
    eng.loop_prepare(labels)
    eng.start_profile(["coda_b200_pi_rank1"])
    for _ in range(3):
        eng.loop_eager()
    prof = eng.stop_profile()
    sel.close()
    assert set(prof) == {"coda_b200_pi_rank1"} and prof["coda_b200_pi_rank1"][0] == 3
