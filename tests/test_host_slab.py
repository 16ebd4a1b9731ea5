"""A host-resident slab (``HostSlab``): CODA, the competing selectors and ``Oracle.true_losses`` on one GPU from an (H, N,
C) slab kept in host memory give the bits of the same slab held as one device tensor; the per-step staging kernel
(``coda_b200_host_stage``) on its own; resume across the two placements; device memory; refusals; main.py through the
shim."""
import ctypes as ct
import io
import random

import numpy as np
import pytest
import torch

from helpers import golden_slab, load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
DTYPES = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
METHODS = {"iid": "IID", "uncertainty": "Uncertainty", "activetesting": "ActiveTesting", "vma": "VMA",
           "model_picker": "ModelPicker"}


def _seed_all(s=0):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)
    torch.cuda.manual_seed_all(s)


def _slab(H, N, C, dtype, seed=3):
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, seed, dtype=DTYPES[dtype])
    return preds.contiguous(), labels


def _ds(preds, labels, host, chunk=None):
    from coda_b200 import HostDataset, HostSlab, TensorDataset
    if host:
        return HostDataset(HostSlab(preds, DEV, chunk_items=chunk), labels.to(DEV))
    return TensorDataset(preds.to(DEV), labels.to(DEV))


def _bits(t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _coda_state(sel):
    return {"D": _bits(sel.dirichlets), "U": _bits(sel.pi_hat_xi), "pi_hat": _bits(sel.pi_hat),
            "pbest": _bits(sel.get_pbest()), "eig": _bits(sel.eig)}


def _same_state(a, b, where):
    for k in a:
        assert torch.equal(a[k], b[k]), (where, k)


def _coda_run(preds, labels, host, *, chunk=None, q="eig", prefilter_n=0, api=3, loop=4, rule="first",
              record_best=True, check=None):
    """``api`` API steps then ``loop`` run_steps steps -> everything compared between the two placements."""
    from coda_b200 import CODA
    _seed_all()
    sel = CODA(_ds(preds, labels, host, chunk), q=q, prefilter_n=prefilter_n)
    states = [_coda_state(sel)] if q == "eig" else []
    trace = []
    for _ in range(api):
        i, qv = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), qv)
        trace.append((int(i), float(qv).hex(), int(sel.get_best_model_prediction())))
        if q == "eig":
            states.append(_coda_state(sel))
    if loop:
        sel.run_steps(loop, labels.to(DEV), record_best=record_best, tie_rule=rule)
    idx, qq, tie = sel.history()
    best, _ = sel.best_history()
    out = {"trace": trace, "states": states, "final": _coda_state(sel), "hist": (idx.tolist(), qq.tobytes(),
           tie.tolist(), best.tolist()), "stochastic": sel.stochastic, "py": random.getstate(),
           "torch": torch.get_rng_state(), "labeled": list(sel.labeled_idxs), "kernels": dict(sel.engine.kernels),
           "n_host": sel.engine.n_host, "host_cols": (int(sel.engine.host_cols.item())
                                                      if sel.engine.host_cols is not None else 0)}
    if check is not None:
        check(sel)
    sel.close()
    return out


def _compare(want, got, where):
    assert want["trace"] == got["trace"], where
    assert len(want["states"]) == len(got["states"])
    for k, (a, b) in enumerate(zip(want["states"], got["states"])):
        _same_state(a, b, (where, "step", k))
    _same_state(want["final"], got["final"], (where, "final"))
    for key in ("hist", "stochastic", "py", "labeled", "kernels"):
        assert want[key] == got[key], (where, key)
    assert torch.equal(want["torch"], got["torch"]), where


# ---------------------------------------------------------------------------------------------------------------------
# CODA, bit for bit against the device-resident run
# ---------------------------------------------------------------------------------------------------------------------
CASES = [
    # (H, N, C, dtype, chunk items, CODA_B200_SHADOW_MODELS, graphs)
    (32, 1001, 10, "f32", 96, "some", True),
    (32, 1001, 10, "f16", 96, "0", False),
    (32, 1001, 10, "bf16", 160, "all", True),
    (1, 777, 3, "f32", 64, "0", True),
    (256, 613, 100, "f32", 256, "some", True),
    (256, 613, 100, "bf16", 96, "0", False),
    (300, 401, 150, "f32", 128, "some", True),
    (300, 401, 150, "f16", 64, "all", False),
]


def _shadow_env(monkeypatch, H, shadow):
    n = {"0": 0, "some": max(0, H // 3), "all": H}[shadow]
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", str(n))
    return n


@pytest.mark.parametrize("H,N,C,dtype,chunk,shadow,graphs", CASES)
def test_coda_host_slab_is_bit_identical(monkeypatch, H, N, C, dtype, chunk, shadow, graphs):
    n_dev = _shadow_env(monkeypatch, H, shadow)
    monkeypatch.setenv("CODA_B200_GRAPH", "1" if graphs else "0")
    preds, labels = _slab(H, N, C, dtype)
    want = _coda_run(preds, labels, False)
    got = _coda_run(preds, labels, True, chunk=chunk)
    _compare(want, got, (H, N, C, dtype, shadow))
    assert got["n_host"] == H - n_dev
    if got["n_host"] and H > 1:
        assert got["host_cols"] > 0                   # some steps did gather host slots


@pytest.mark.parametrize("q,prefilter_n,rule", [("eig", 0, "reference"), ("eig", 50, "first"), ("eig", 50, "reference"),
                                                ("iid", 0, "first"), ("uncertainty", 0, "first"),
                                                ("uncertainty", 0, "reference")])
def test_coda_host_slab_every_acquisition(monkeypatch, q, prefilter_n, rule):
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "7")
    preds, labels = _slab(24, 903, 12, "f32", seed=11)
    want = _coda_run(preds, labels, False, q=q, prefilter_n=prefilter_n, rule=rule, api=2, loop=5)
    got = _coda_run(preds, labels, True, chunk=224, q=q, prefilter_n=prefilter_n, rule=rule, api=2, loop=5)
    _compare(want, got, (q, prefilter_n, rule))


@pytest.mark.parametrize("name", ["traj_small_h32_n3000_c10", "traj_h256_h256_n1500_c100"])
def test_reference_goldens_through_host_slab(monkeypatch, name):
    """The reference's trajectory, teacher-forced, under the tolerances of test_gpu_parity, with half the models in
    host slots."""
    from coda_b200 import CODA, HostDataset, HostSlab
    g = load_golden(name)
    preds, labels = golden_slab(g)
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", str(int(g["H"]) // 2))
    random.seed(0)
    sel = CODA(HostDataset(HostSlab(preds.contiguous(), DEV, chunk_items=int(g["N"]) // 3), labels.to(DEV)),
               **g["ctor"])
    assert sel.engine.n_host == int(g["H"]) - int(g["H"]) // 2
    if "init_dirichlets" in g:
        np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), g["init_dirichlets"], rtol=2e-6, atol=1e-7)
    np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), g["init_pi_hat"], rtol=2e-6)
    for k in range(int(g["steps"])):
        idx, q = sel.get_next_item_to_label()
        ref = g["eig"][k]
        cand = ~np.isnan(ref)
        np.testing.assert_allclose(sel.engine.eig.cpu().numpy()[cand], ref[cand], atol=5e-6)
        gi = int(g["idx"][k])                     # teacher forcing: follow the reference's pick
        t = int(labels[gi])
        sel.add_label(gi, t, q)
        assert int(sel.get_best_model_prediction()) == int(g["best_model"][k])
        np.testing.assert_allclose(sel.get_pbest().cpu().numpy()[0], g["pbest"][k], atol=1e-5)
        np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), g["pi_hat"][k], rtol=2e-6)
        np.testing.assert_allclose(sel.dirichlets[:, t].cpu().numpy(), g["dir_row"][k], rtol=3e-7, atol=0)
    assert int(sel.engine.host_cols.item()) > 0
    sel.close()


# ---------------------------------------------------------------------------------------------------------------------
# the competing selectors
# ---------------------------------------------------------------------------------------------------------------------
def _bl_run(method, preds, labels, host, chunk=None, api=4, loop=6, rule="philox"):
    import coda_b200
    from coda.options import LOSS_FNS
    _seed_all()
    ds = _ds(preds, labels, host, chunk)
    cls = getattr(coda_b200, METHODS[method])
    sel = cls(ds) if method == "model_picker" else cls(ds, LOSS_FNS["acc"])
    trace = []
    for _ in range(api):
        i, qv = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), qv)
        trace.append((int(i), float(qv).hex(), int(sel.get_best_model_prediction())))
    if rule == "philox":
        sel.run_steps(loop, labels.to(DEV), seed=5)
    else:
        sel.run_steps(loop, labels.to(DEV), tie_rule="reference")
    idx, q, tie = sel.history()
    best, btie = sel.best_history()
    out = {"trace": trace, "hist": (idx.tolist(), q.tobytes(), tie.tolist(), best.tolist(), btie.tolist()),
           "stochastic": sel.stochastic, "py": random.getstate(), "torch": torch.get_rng_state(),
           "cuda": torch.cuda.get_rng_state(DEV)}
    sel.close()
    return out


@pytest.mark.parametrize("method", list(METHODS))
@pytest.mark.parametrize("dtype,rule", [("f32", "philox"), ("bf16", "reference"), ("f16", "philox")])
def test_competing_selectors_host_slab_are_bit_identical(method, dtype, rule):
    preds, labels = _slab(20, 517, 7, dtype, seed=5)
    want = _bl_run(method, preds, labels, False, rule=rule)
    got = _bl_run(method, preds, labels, True, chunk=96, rule=rule)
    for k in ("trace", "hist", "stochastic", "py"):
        assert want[k] == got[k], (method, dtype, k)
    assert torch.equal(want["torch"], got["torch"]) and torch.equal(want["cuda"], got["cuda"])


# ---------------------------------------------------------------------------------------------------------------------
# resume across the two placements
# ---------------------------------------------------------------------------------------------------------------------
def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=False)


@pytest.mark.parametrize("first_host", [False, True])
def test_coda_resume_across_placements(monkeypatch, first_host):
    from coda_b200 import CODA
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "5")
    preds, labels = _slab(16, 611, 9, "f32", seed=8)
    lab = labels.to(DEV)

    def steps(sel, k):
        out = []
        for _ in range(k):
            i, qv = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), qv)
            out.append((int(i), float(qv).hex()))
        return out
    _seed_all()
    ref = CODA(_ds(preds, labels, False))
    want = steps(ref, 3)
    ref.run_steps(4, lab)
    want_hist = ref.history()[0].tolist()
    want_state = _coda_state(ref)
    ref.close()
    _seed_all()
    a = CODA(_ds(preds, labels, first_host, 128))
    got = steps(a, 3)
    sd = _roundtrip(a.state_dict())
    a.close()
    random.seed(99)
    b = CODA(_ds(preds, labels, not first_host, 128))
    b.load_state_dict(sd)
    b.run_steps(4, lab)
    assert got == want
    assert b.history()[0].tolist()[-4:] == want_hist[-4:]
    _same_state(want_state, _coda_state(b), "resumed")
    b.close()


@pytest.mark.parametrize("method", ["activetesting", "model_picker"])
def test_competing_selector_resume_across_placements(method):
    import coda_b200
    from coda.options import LOSS_FNS
    preds, labels = _slab(12, 400, 5, "f32", seed=2)
    lab = labels.to(DEV)

    def make(host):
        cls = getattr(coda_b200, METHODS[method])
        ds = _ds(preds, labels, host, 96)
        return cls(ds) if method == "model_picker" else cls(ds, LOSS_FNS["acc"])

    for first_host in (False, True):
        _seed_all()
        ref = make(False)
        ref.run_steps(8, lab, seed=3)
        want = ref.history()[0].tolist()
        ref.close()
        _seed_all()
        a = make(first_host)
        a.run_steps(3, lab, seed=3)
        sd = _roundtrip(a.state_dict())
        a.close()
        b = make(not first_host)
        b.load_state_dict(sd)
        b.run_steps(5, lab, seed=3)
        got = b.history()[0].tolist()
        b.close()
        assert len(got) == 8 and got[:3] == want[:3], (method, first_host)


# ---------------------------------------------------------------------------------------------------------------------
# the staging kernel alone
# ---------------------------------------------------------------------------------------------------------------------
def _stage_case(H, dtype, seed, host_share):
    """A teacher-forced gather list over a fake host-mode layout -> (step struct, buffers, expected)."""
    from coda_b200 import _native as nat
    from coda_b200.engine import _PinnedHost
    lib = nat.load()
    g = torch.Generator().manual_seed(seed)
    C, N = 5, 203
    dt = DTYPES[dtype]
    esz = torch.empty(0, dtype=dt).element_size()
    cs = (N + 7) // 8 * 8 if esz == 2 else (N + 3) // 4 * 4
    S = int(H * (1 - host_share))
    nh = H - S
    hs = _PinnedHost((max(1, nh), C, cs), dt, lib)
    hs.t.copy_(torch.rand((max(1, nh), C, cs), generator=g).to(dt))
    stage = torch.full((2 * max(1, nh) * cs,), float("nan"), dtype=dt, device=DEV)
    base = stage.data_ptr() - 4096 * 16                      # any slab base; the staging offset is relative to it
    stage_off = (stage.data_ptr() - base) // esz
    terms, want = [], []
    if H > 1:
        terms.append((1234, 1.0, 1))                          # the ensemble term
    r = 0
    for h in range(H):
        j, tp = int(torch.randint(C, (1,), generator=g)), int(torch.randint(C, (1,), generator=g))
        two = bool(torch.randint(2, (1,), generator=g))
        for c, sg in ([(j, 1.0), (tp, -1.0)] if two else [(j, 1.0)]):
            if h >= S:
                off = ((h - S) * C + c) * cs
                terms.append((off, sg, 0))
                want.append((stage_off + r * cs, sg, 1, off))
                r += 1
            else:
                terms.append((h * 1000 + c * 7, sg, 1 if h % 2 else C))
                want.append(None)
    nt = len(terms)
    buf = torch.zeros(2 + 4 * (2 * H + 2), dtype=torch.int32)
    buf[0], buf[1] = nt, 3
    raw = buf.numpy()
    for k, (off, sg, st) in enumerate(terms):
        b = 2 + 4 * k
        raw[b:b + 2] = np.array([off], dtype=np.int64).view(np.int32)
        raw[b + 2] = np.array([sg], dtype=np.float32).view(np.int32)[0]
        raw[b + 3] = st
    terms_dev = torch.zeros(len(raw) // 2 + 1, dtype=torch.int64, device=DEV).view(torch.int32)[:len(raw)]
    terms_dev.copy_(buf)
    st = nat.StepStruct()
    st.H, st.C, st.N = H, C, N
    st.terms = terms_dev.data_ptr()
    st.shadow_col_stride = cs
    st.n_host, st.host_shadow, st.stage, st.stage_off = nh, hs.data_ptr(), stage.data_ptr(), stage_off
    st.flags = 0
    return lib, nat, st, terms_dev, buf, terms, want, hs, stage, cs, esz


def _decode(t):
    a = t.cpu().numpy()
    out = []
    for k in range(int(a[0])):
        b = 2 + 4 * k
        out.append((int(a[b:b + 2].view(np.int64)[0]), float(a[b + 2:b + 3].view(np.float32)[0]), int(a[b + 3])))
    return out


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("H,host_share", [(1, 1.0), (9, 0.5), (256, 0.3), (1024, 0.9), (64, 0.0)])
def test_host_stage_kernel(dtype, H, host_share):
    lib, nat, st, terms_dev, buf, terms, want, hs, stage, cs, esz = _stage_case(H, dtype, H + len(dtype), host_share)
    census = torch.zeros(1, dtype=torch.int64, device=DEV)
    before = terms_dev.clone()
    nat.check(lib.coda_b200_host_stage(ct.byref(st), nat.slab_format(DTYPES[dtype]), ct.c_void_p(census.data_ptr()),
                                       ct.c_void_p(torch.cuda.current_stream(DEV).cuda_stream)), "host_stage")
    torch.cuda.synchronize()
    got = _decode(terms_dev)
    assert len(got) == len(terms) and int(terms_dev[1]) == 3
    hostflat = hs.t.reshape(-1)
    nh = sum(1 for w in want if w is not None)
    assert int(census.item()) == (nh if st.n_host else 0)
    k0 = len(terms) - len(want)
    for k, (g, t) in enumerate(zip(got, terms)):
        assert g[1] == t[1], k                                # signs and order unchanged
        w = want[k - k0] if k >= k0 else None
        if w is None:
            assert g == t, k                                  # device terms untouched
        else:
            assert g == w[:3], k
            col = stage[w[0] - st.stage_off: w[0] - st.stage_off + cs].cpu()
            assert torch.equal(col.view(torch.int16 if esz == 2 else torch.int32),
                               hostflat[w[3]: w[3] + cs].view(torch.int16 if esz == 2 else torch.int32)), k
    if nh == 0:
        assert torch.equal(terms_dev, before) and bool(torch.isnan(stage.float()).all())


# ---------------------------------------------------------------------------------------------------------------------
# Oracle, memory, refusals, the shim
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", list(DTYPES))
def test_oracle_true_losses_host_slab(dtype):
    from coda.options import LOSS_FNS
    from coda_b200 import HostDataset, HostSlab, Oracle, TensorDataset
    preds, labels = _slab(11, 1003, 13, dtype)
    want = Oracle(TensorDataset(preds.to(DEV), labels.to(DEV)), LOSS_FNS["acc"])
    want = want.true_losses(want.dataset.preds)
    ds = HostDataset(HostSlab(preds, DEV, chunk_items=200), labels.to(DEV))
    got = Oracle(ds, LOSS_FNS["acc"]).true_losses(ds.preds)
    assert torch.equal(_bits(want), _bits(got))


def test_device_memory_stays_within_state_chunk_and_staging(monkeypatch):
    """The slab (768 MB) is most of the figure: a device-resident slab would exceed the bound."""
    from coda_b200 import CODA, HostDataset, HostSlab
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "2")
    H, N, C = 96, 200000, 10
    preds, labels = _slab(H, N, C, "f32")
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    slab = HostSlab(preds, DEV, chunk_items=8192)
    sel = CODA(HostDataset(slab, labels.to(DEV)))
    e = sel.engine
    for _ in range(2):
        i, qv = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), qv)
    sel.run_steps(3, labels.to(DEV))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV) - base
    state = sum(v.numel() * v.element_size() for v in e.__dict__.values()
                if isinstance(v, torch.Tensor) and v.is_cuda and v._base is None)
    from coda_b200.datasets import DEFAULT_CHUNK_BYTES
    bound = state + 2 * slab.chunk_bytes() + DEFAULT_CHUNK_BYTES + (64 << 20)    # + construction temporaries
    assert peak <= bound, (peak, state, slab.chunk_bytes())
    assert peak < preds.numel() * 4                            # the slab itself never sat on the device
    hs = e.host_slots
    assert hs is not None
    sel.close()
    assert e.host_slots is None


def test_refusals_raise_before_launching(monkeypatch):
    from coda_b200 import CODA, IID, HostDataset, HostSlab
    from coda.options import LOSS_FNS
    from coda_b200.eps_search import modelpicker_eps_search
    preds, labels = _slab(8, 300, 4, "f32")
    ds = HostDataset(HostSlab(preds, DEV), labels.to(DEV))
    for kw in ({"gpus": 2}, {"shards": 2}):
        with pytest.raises(NotImplementedError):
            CODA(ds, **kw)
        with pytest.raises(NotImplementedError):
            IID(ds, LOSS_FNS["acc"], **kw)
    with pytest.raises(NotImplementedError):
        CODA(ds, mode="recompute_all")
    with pytest.raises(NotImplementedError):
        modelpicker_eps_search(ds, [0.5], iterations=1, pool_size=4, budget=2, seed=0)


def test_main_py_cfg1_under_host_slab(tmp_path):
    import test_main_py_cfg1 as m
    (tmp_path / "dev").mkdir()
    (tmp_path / "host").mkdir()
    _g, dev_out, _ = m._run(tmp_path / "dev", iters=12)
    _g, host_out, stdout = m._run(tmp_path / "host", extra_env={"CODA_B200_HOST_SLAB": "1"}, iters=12)
    for k in ("chosen_idx", "true_class", "best_model", "regret", "cumulative_regret"):
        assert dev_out[k] == host_out[k], k
