"""A host-resident slab in N-range pieces (``ShardedHostSlab``): CODA, the competing selectors and
``Oracle.true_losses`` on host pieces give the bits of the same ranges held as device pieces (``ShardedSlab``), of one
``HostSlab`` and of the plain tensor; checkpoints cross the layouts; the loader and device memory; refusals.  All pieces
share this GPU, as in test_sharding.py."""
import io
import random

import numpy as np
import pytest
import torch

from helpers import golden_slab, load_golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
METHODS = {"iid": "IID", "uncertainty": "Uncertainty", "activetesting": "ActiveTesting", "vma": "VMA",
           "model_picker": "ModelPicker"}


def _seed_all(s=0):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)
    torch.cuda.manual_seed_all(s)


def _bits(t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _cuts(N, k):
    """Uneven N-ranges: piece r holds about (r + 1) shares."""
    w = [r + 1 for r in range(k)]
    ends = [N * sum(w[:r + 1]) // sum(w) for r in range(k)]
    return list(zip([0] + ends[:-1], ends))


def _ds(preds, labels, layout, k=1, dtype=None, chunk=None):
    """``preds`` (CPU) held as ``layout``: 'tensor', 'host' (one HostSlab), 'dev_pieces' (ShardedSlab) or 'host_pieces'
    (ShardedHostSlab of N-range views of ``preds``), read at ``dtype`` (default: the tensor's own)."""
    from coda_b200 import HostDataset, HostSlab, ShardedHostSlab, ShardedSlab, TensorDataset
    dtype = dtype or preds.dtype
    lab = labels.to(DEV)
    if layout == "tensor":
        return TensorDataset(preds.to(dtype).to(DEV), lab)
    if layout == "host":
        return HostDataset(HostSlab(preds, DEV, dtype=dtype, chunk_items=chunk), lab)
    if layout == "dev_pieces":
        return TensorDataset(ShardedSlab([preds[:, lo:hi].to(dtype).contiguous().to(DEV) for lo, hi in _cuts(
            preds.shape[1], k)]), lab)
    s = ShardedHostSlab([HostSlab(preds[:, lo:hi], DEV, dtype=dtype, chunk_items=chunk)
                         for lo, hi in _cuts(preds.shape[1], k)])
    assert all(p.host.untyped_storage().data_ptr() == preds.untyped_storage().data_ptr() for p in s.pieces)
    return TensorDataset(s, lab)


def _coda_state(sel, eig=True):
    out = {"D": _bits(sel.dirichlets), "U": _bits(sel.pi_hat_xi), "pi_hat": _bits(sel.pi_hat),
           "pbest": _bits(sel.get_pbest())}
    if eig:
        out["eig"] = _bits(sel.eig)
    return out


def _coda_run(ds, labels, *, q="eig", prefilter_n=0, api=3, loop=4, rule="first"):
    from coda_b200 import CODA
    _seed_all()
    sel = CODA(ds, q=q, prefilter_n=prefilter_n)
    eig = q == "eig" and not prefilter_n               # a prefilter_n pass scores only its sample
    states = [_coda_state(sel, eig)]
    trace = []
    for _ in range(api):
        i, qv = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), qv)
        trace.append((int(i), float(qv).hex(), int(sel.get_best_model_prediction())))
        states.append(_coda_state(sel, eig))
    sel.run_steps(loop, labels.to(DEV), record_best=True, tie_rule=rule)
    idx, qq, tie = sel.history()
    best, _ = sel.best_history()
    out = {"trace": trace, "states": states, "final": _coda_state(sel, eig),
           "hist": (idx.tolist(), qq.tobytes(), tie.tolist(), best.tolist()), "stochastic": sel.stochastic,
           "py": random.getstate(), "torch": torch.get_rng_state(), "labeled": list(sel.labeled_idxs),
           "kernels": [dict(e.kernels) for e in sel.engines], "n_host": [e.n_host for e in sel.engines],
           "S": [e.n_shadow for e in sel.engines],
           "host_cols": [int(e.host_cols.item()) if e.host_cols is not None else 0 for e in sel.engines]}
    sel.close()
    return out


def _compare(want, got, where):
    assert want["trace"] == got["trace"], where
    assert len(want["states"]) == len(got["states"])
    for k, (a, b) in enumerate(zip(want["states"], got["states"])):
        for key in a:
            assert torch.equal(a[key], b[key]), (where, "step", k, key)
    for key in want["final"]:
        assert torch.equal(want["final"][key], got["final"][key]), (where, "final", key)
    for key in ("hist", "stochastic", "py", "labeled"):
        assert want[key] == got[key], (where, key)
    assert torch.equal(want["torch"], got["torch"]), where


# ---------------------------------------------------------------------------------------------------------------------
# CODA, bit for bit against device pieces, one HostSlab and the plain tensor
# ---------------------------------------------------------------------------------------------------------------------
CASES = [
    # (pieces, H, N, C, stored dtype, read as, chunk items, graphs)
    (2, 32, 1001, 10, torch.float32, torch.float32, 96, True),
    (3, 32, 1001, 10, torch.float16, torch.float16, 64, False),
    (3, 32, 1001, 10, torch.float16, torch.float32, 160, True),
    (2, 256, 613, 100, torch.float32, torch.float32, 96, False),
    (3, 48, 2003, 16, torch.float16, torch.float32, 128, False),
]


@pytest.mark.parametrize("k,H,N,C,stored,read,chunk,graphs", CASES)
def test_coda_host_pieces_are_bit_identical(monkeypatch, k, H, N, C, stored, read, chunk, graphs):
    from coda_b200.synth import synth
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", str(H // 3))          # every piece keeps host slots
    monkeypatch.setenv("CODA_B200_GRAPH", "1" if graphs else "0")
    preds, labels = synth(H, N, C, 3, dtype=stored)
    preds = preds.contiguous()
    assert all(chunk < hi - lo for lo, hi in _cuts(N, k))                # every walk takes several chunks
    got = _coda_run(_ds(preds, labels, "host_pieces", k, read, chunk), labels)
    assert got["n_host"] == [H - H // 3] * k and got["S"] == [H // 3] * k
    assert all(c > 0 for c in got["host_cols"]), got["host_cols"]        # every piece staged host columns
    pieces = _coda_run(_ds(preds, labels, "dev_pieces", k, read), labels)
    _compare(pieces, got, "device pieces")
    assert pieces["kernels"] == got["kernels"]                           # each piece took the kernels its twin took
    _compare(_coda_run(_ds(preds, labels, "host", 1, read, chunk), labels), got, "one HostSlab")
    _compare(_coda_run(_ds(preds, labels, "tensor", 1, read), labels), got, "tensor")


@pytest.mark.parametrize("q,prefilter_n,rule", [("eig", 0, "reference"), ("eig", 50, "first"), ("eig", 50, "reference"),
                                                ("iid", 0, "first"), ("iid", 0, "reference"),
                                                ("uncertainty", 0, "first"), ("uncertainty", 0, "reference")])
def test_coda_host_pieces_every_acquisition(monkeypatch, q, prefilter_n, rule):
    from coda_b200.synth import synth
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "7")
    preds, labels = synth(24, 903, 12, 11)
    preds = preds.contiguous()
    kw = dict(q=q, prefilter_n=prefilter_n, rule=rule, api=2, loop=5)
    got = _coda_run(_ds(preds, labels, "host_pieces", 3, chunk=96), labels, **kw)
    _compare(_coda_run(_ds(preds, labels, "dev_pieces", 3), labels, **kw), got, "device pieces")
    _compare(_coda_run(_ds(preds, labels, "tensor"), labels, **kw), got, "tensor")


def test_coda_host_pieces_reference_ties(monkeypatch):
    """traj_tiny's items three times over: exact EIG ties every step, the copies on different pieces."""
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "3")
    g = load_golden("traj_tiny_h8_n300_c5")
    preds, labels = golden_slab(g)
    order = torch.arange(preds.shape[1]).repeat(3)
    preds, labels = preds[:, order].contiguous(), labels[order].contiguous()
    got = _coda_run(_ds(preds, labels, "host_pieces", 3, chunk=64), labels, api=2, loop=10, rule="reference")
    assert sum(got["hist"][2]) >= 3
    _compare(_coda_run(_ds(preds, labels, "dev_pieces", 3), labels, api=2, loop=10, rule="reference"), got, "pieces")
    _compare(_coda_run(_ds(preds, labels, "tensor"), labels, api=2, loop=10, rule="reference"), got, "tensor")


def test_reference_golden_trajectory_on_host_pieces(monkeypatch):
    """The reference's free-running trajectory from host pieces, under test_sharding's tolerances."""
    from coda_b200 import CODA
    g = load_golden("traj_small_h32_n3000_c10")
    preds, labels = golden_slab(g)
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "10")
    sel = CODA(_ds(preds.contiguous(), labels, "host_pieces", 3, chunk=256))
    assert len(sel.engines) == 3 and all(e.n_host == 22 for e in sel.engines)
    np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), g["init_pi_hat"], rtol=2e-6)
    sel.run_steps(int(g["steps"]), labels.to(DEV))
    idx, q, tie = sel.history()
    assert idx.tolist() == [int(i) for i in g["idx"]] and not tie.any()
    np.testing.assert_allclose(q, g["q"], atol=5e-6)
    np.testing.assert_allclose(sel.get_pbest().cpu().numpy()[0], g["pbest"][-1], atol=1e-5)
    np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), g["final_dirichlets"], rtol=2e-6, atol=1e-7)
    assert all(int(e.host_cols.item()) > 0 for e in sel.engines)
    sel.close()


# ---------------------------------------------------------------------------------------------------------------------
# the competing selectors
# ---------------------------------------------------------------------------------------------------------------------
def _bl_run(method, ds, labels, api=4, loop=6, rule="philox"):
    import coda_b200
    from coda.options import LOSS_FNS
    _seed_all()
    cls = getattr(coda_b200, METHODS[method])
    sel = cls(ds) if method == "model_picker" else cls(ds, LOSS_FNS["acc"])
    trace = [int(sel.get_best_model_prediction())]
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
           "stochastic": sel.stochastic, "py": random.getstate(), "torch": torch.get_rng_state().numpy().tobytes(),
           "cuda": torch.cuda.get_rng_state(DEV).numpy().tobytes(), "shards": len(sel.states)}
    sel.close()
    return out


@pytest.mark.parametrize("method", list(METHODS))
@pytest.mark.parametrize("rule", ["philox", "reference"])
def test_competing_selectors_on_host_pieces_equal_device_pieces(method, rule):
    from coda_b200.synth import synth
    preds, labels = synth(20, 517, 7, 5)
    preds = preds.contiguous()
    for k, stored in ((2, torch.float32), (3, torch.bfloat16)):
        p = preds.to(stored)
        want = _bl_run(method, _ds(p, labels, "dev_pieces", k), labels, rule=rule)
        got = _bl_run(method, _ds(p, labels, "host_pieces", k, chunk=64), labels, rule=rule)
        assert got["shards"] == k
        for key in want:
            assert want[key] == got[key], (method, rule, k, key)


# ---------------------------------------------------------------------------------------------------------------------
# checkpoints across the layouts
# ---------------------------------------------------------------------------------------------------------------------
def _roundtrip(sd):
    buf = io.BytesIO()
    torch.save(sd, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=False)


@pytest.mark.parametrize("first,second", [("host_pieces", "dev_pieces"), ("host_pieces", "host"),
                                          ("dev_pieces", "host_pieces"), ("host", "host_pieces")])
def test_coda_resume_across_layouts(monkeypatch, first, second):
    from coda_b200 import CODA
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "5")
    from coda_b200.synth import synth
    preds, labels = synth(16, 611, 9, 8)
    preds = preds.contiguous()
    lab = labels.to(DEV)

    def steps(sel, k):
        out = []
        for _ in range(k):
            i, qv = sel.get_next_item_to_label()
            sel.add_label(i, int(labels[i]), qv)
            out.append((int(i), float(qv).hex()))
        return out
    _seed_all()
    ref = CODA(_ds(preds, labels, "tensor"))
    want = steps(ref, 3)
    ref.run_steps(4, lab)
    want_hist = ref.history()[0].tolist()[-4:]
    want += steps(ref, 2)
    want_state = _coda_state(ref)
    ref.close()
    _seed_all()
    a = CODA(_ds(preds, labels, first, 3, chunk=96))
    got = steps(a, 3)
    sd = _roundtrip(a.state_dict())
    a.close()
    random.seed(99)
    b = CODA(_ds(preds, labels, second, 2, chunk=128))
    b.load_state_dict(sd)
    b.run_steps(4, lab)
    assert b.history()[0].tolist()[-4:] == want_hist
    got += steps(b, 2)
    assert got == want
    state = _coda_state(b)
    for key in want_state:
        assert torch.equal(want_state[key], state[key]), key
    b.close()


@pytest.mark.parametrize("method", ["activetesting", "model_picker"])
def test_competing_selector_resume_across_layouts(method):
    import coda_b200
    from coda.options import LOSS_FNS
    from coda_b200.synth import synth
    preds, labels = synth(12, 400, 5, 2)
    preds = preds.contiguous()
    lab = labels.to(DEV)

    def make(layout, k):
        cls = getattr(coda_b200, METHODS[method])
        ds = _ds(preds, labels, layout, k, chunk=64)
        return cls(ds) if method == "model_picker" else cls(ds, LOSS_FNS["acc"])

    _seed_all()
    ref = make("tensor", 1)
    ref.run_steps(8, lab, seed=3)
    want = ref.history()[0].tolist()
    ref.close()
    for first, second in (("host_pieces", "dev_pieces"), ("dev_pieces", "host_pieces"), ("host_pieces", "host"),
                          ("host", "host_pieces")):
        _seed_all()
        a = make(first, 3)
        a.run_steps(3, lab, seed=3)
        sd = _roundtrip(a.state_dict())
        a.close()
        b = make(second, 2)
        b.load_state_dict(sd)
        b.run_steps(5, lab, seed=3)
        got = b.history()[0].tolist()
        b.close()
        assert len(got) == 8 and got[:3] == want[:3], (method, first, second)


# ---------------------------------------------------------------------------------------------------------------------
# Oracle, loader, memory, refusals
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stored,read", [(torch.float32, torch.float32), (torch.float16, torch.float16),
                                         (torch.bfloat16, torch.float32)])
def test_oracle_true_losses_on_host_pieces(stored, read):
    from coda.options import LOSS_FNS
    from coda_b200 import Oracle
    from coda_b200.synth import synth
    preds, labels = synth(11, 1003, 13, 3, dtype=stored)
    preds = preds.contiguous()
    want = Oracle(_ds(preds, labels, "tensor", dtype=read), LOSS_FNS["acc"])
    want = want.true_losses(want.dataset.preds)
    for k in (2, 3):
        ds = _ds(preds, labels, "host_pieces", k, read, chunk=96)
        got = Oracle(ds, LOSS_FNS["acc"]).true_losses(ds.preds)
        assert got.device == want.device and torch.equal(_bits(want), _bits(got)), k


@pytest.mark.parametrize("keep", [False, True])
def test_loaded_host_pieces_stream_what_load_sharded_holds(tmp_path, keep):
    """Each piece's walk hands its kernels the bytes of load_sharded's piece; CODA on the loaded host pieces follows
    CODA on the loaded device pieces."""
    from coda_b200 import CODA
    from coda_b200.datasets import Dataset, ShardedHostSlab, load_host, load_sharded
    H, N, C = 6, 1003, 7
    t = torch.rand(H, N, C, generator=torch.Generator().manual_seed(1)).softmax(-1).to(torch.float16)
    p = str(tmp_path / "task.pt")
    torch.save(t, p)
    torch.save(torch.randint(0, C, (N,)), p.replace(".pt", "_labels.pt"))
    dev = load_sharded(p, DEV, keep, shards=3, gpus=1)
    host = load_host(p, DEV, keep, shards=3, gpus=1, chunk_items=64)
    assert isinstance(host, ShardedHostSlab) and host.offsets == dev.offsets and host.dtype == dev.dtype
    for hp, dp in zip(host.pieces, dev.pieces):
        assert hp.device == dp.device
        seen = []
        hp.walk(lambda n0, n1, v: seen.append((n0, v.clone())))
        assert len(seen) > 1
        for n0, v in seen:
            assert torch.equal(v.view(torch.uint8), dp[:, n0:n0 + v.shape[1]].contiguous().view(torch.uint8))
        for i in (0, int(hp.shape[1]) - 1):
            assert torch.equal(hp.item_column(i), dp[:, i].float())
    runs = []
    for kw in ({"host": True}, {}):
        ds = Dataset(p, DEV, keep_dtype=keep, shards=3, gpus=1, **kw)
        random.seed(0)
        sel = CODA(ds)
        for _ in range(3):
            i, q = sel.get_next_item_to_label()
            sel.add_label(i, int(ds.labels[i]), q)
        sel.run_steps(4, ds.labels)
        runs.append((sel.history()[0].tolist(), sel.history()[1].tobytes(), _coda_state(sel)))
        sel.close()
    assert runs[0][:2] == runs[1][:2]
    for key in runs[0][2]:
        assert torch.equal(runs[0][2][key], runs[1][2][key]), key


def test_device_memory_stays_within_the_pieces_state_chunks_and_staging(monkeypatch):
    """Two host pieces on this GPU: the slab (768 MB) never sits on the device; the peak is the pieces' state plus one
    walk's chunk buffers (construction walks one piece at a time) and the widening chunk."""
    from coda_b200 import CODA
    from coda_b200.datasets import DEFAULT_CHUNK_BYTES
    from coda_b200.synth import synth
    monkeypatch.setenv("CODA_B200_SHADOW_MODELS", "2")
    H, N, C = 96, 200000, 10
    preds, labels = synth(H, N, C, 3)
    preds = preds.contiguous()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    ds = _ds(preds, labels, "host_pieces", 2, chunk=8192)
    sel = CODA(ds)
    for _ in range(2):
        i, qv = sel.get_next_item_to_label()
        sel.add_label(i, int(labels[i]), qv)
    sel.run_steps(3, labels.to(DEV))
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV) - base
    state = sum(v.numel() * v.element_size() for e in sel.engines for v in e.__dict__.values()
                if isinstance(v, torch.Tensor) and v.is_cuda and v._base is None)
    chunks = max(2 * p.chunk_bytes() for p in ds.preds.pieces)
    bound = state + N * 8 + chunks + DEFAULT_CHUNK_BYTES + (64 << 20)    # + labels, construction temporaries
    assert peak <= bound, (peak, state, chunks)
    assert peak < preds.numel() * 4
    assert all(e.host_slots is not None for e in sel.engines)
    engines = list(sel.engines)
    sel.close()
    assert all(e.host_slots is None for e in engines)


class _World2:
    world, rank = 2, 0


def test_refusals_raise_before_launching(monkeypatch):
    from coda.options import LOSS_FNS
    from coda_b200 import CODA, IID, ModelPicker
    from coda_b200.eps_search import modelpicker_eps_search
    from coda_b200.synth import synth
    preds, labels = synth(8, 300, 4, 3)
    ds = _ds(preds.contiguous(), labels, "host_pieces", 2)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(DEV)
    makers = (lambda **kw: CODA(ds, **kw), lambda **kw: IID(ds, LOSS_FNS["acc"], **kw),
              lambda **kw: ModelPicker(ds, **kw))
    for make in makers:
        for kw in ({"gpus": 3}, {"shards": 3}, {"shards": 2, "gpus": 2}):
            with pytest.raises(ValueError, match="disagrees"):
                make(**kw)
        with pytest.raises(ValueError, match="torch.distributed"):
            make(comm=_World2())
    with pytest.raises(NotImplementedError, match="recompute_all"):
        CODA(ds, mode="recompute_all")
    with pytest.raises(NotImplementedError, match="ShardedHostSlab"):
        modelpicker_eps_search(ds, [0.5], iterations=1, pool_size=4, budget=2, seed=0)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated(DEV) == before
    sel = CODA(ds, shards=2, gpus=1)                                   # the layout the pieces are
    assert len(sel.engines) == 2
    sel.close()
