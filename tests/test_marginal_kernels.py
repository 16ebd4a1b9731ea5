"""Kernel-level tier of the state every EIG is weighted by: the slab scan, the confusion sums, the Dirichlet prior, the
row normalisation with its fixed-point column sums, the posterior update with its gather list and the rank-1 marginal
refresh, each against a host model of that one stage evaluated on the exact inputs the stage received (the engine's own
slab, pseudo labels, D, U, jvec, sel and gather list, copied out before the launch).

  scan       coda_b200_scan_slab(_x)          hard, disagree, E, pseudo, flag bits              (slab.cu)
  confusion  coda_b200_confusion_sorted/accum  int64 fixed-point sums, bit for bit               (slab.cu)
  prior      coda_b200_init_dirichlets         fp64 restatement of coda.py:43-63, 196             (slab.cu)
  normalise  coda_b200_pi_reduce               xi and the column sums, these bit for bit          (slab.cu)
  label      coda_b200_step_label              D, jvec, pisum and the decoded gather list         (step.cu)
  rank-1     coda_b200_pi_rank1(_x)            column t against fp64, every other column's bits   (slab.cu)
  long run   the host-free loop, 1 200 labels  U and pi_hat_xi against fp64 on the final D
  C = 4096   construction and steps at the documented class count, against the oracle

The full pass (pi_full, SIMT and tensor core) is checked against fp64 in test_gpu_parity.py::
test_tensor_core_marginals_match_fp64.  Outputs are filled with NaN (integers: a poison pattern) before each launch,
the path that ran is asserted, and every stage shows once that its comparison fails on a perturbed model.  The CPU
tests at the top anchor the host models to the reference's goldens and the oracle.  Run with ``-s`` to see the worst
error of every comparison against its bound."""
import contextlib
import math
import os

import numpy as np
import pytest
import torch

from helpers import coda_oracle, golden_names, golden_slab, load_golden

U32 = 2.0 ** -24                         # fp32 unit roundoff
NAN = float("nan")
POISON = -0x5A5A5A5B                     # int32 / int64 outputs are filled with this before a launch


def _report(stage, label, err, tol):
    print(f"[marginal] {stage:<9} {label:<44} worst {err:.3e}   bound {tol:.1e}")


# ------------------------------------------------------------------------------------------------------------------
# host models
# ------------------------------------------------------------------------------------------------------------------
def fx_shift_of(n_global):
    """Engine.fx_shift: N_global * 2^shift < 2^62."""
    return max(8, min(40, 62 - math.ceil(math.log2(n_global + 1))))


def scan_model(p32, first=True):
    """(H, N, C) fp32 slab -> hard (N, H), disagree (N,), E (N, C) fp32 summed in model order, pseudo (N,).
    Arg-max takes the first index among equal values (torch.argmax, coda.py:194); ``first=False`` the last one."""
    H = p32.shape[0]
    E = np.zeros(p32.shape[1:], np.float32)
    for h in range(H):
        E += p32[h]                                                      # fp32, h = 0 ... H - 1
    am = (lambda a: a.argmax(-1)) if first else (lambda a: a.shape[-1] - 1 - a[..., ::-1].argmax(-1))
    hard = am(p32).T
    pseudo = am(E / np.float32(H))
    return hard, (hard != hard[:, :1]).any(1), E, pseudo


def confusion_model(p32, pseudo, shift, C, rnd=np.rint):
    """sum_{n: pseudo_n = y} rint(preds * 2^s) in int64: p * 2^s is exact in fp32 and fp64, rint rounds half to even as
    __float2ll_rn does."""
    q = rnd(p32.astype(np.float64) * 2.0 ** shift).astype(np.int64)
    out = np.zeros((p32.shape[0], C, C), np.int64)
    for y in np.unique(pseudo):
        out[:, y] = q[:, pseudo == y].sum(1)
    return out


def prior_model(conf_fx, shift, prior_strength, multiplier, uniform, rest=None, off=None):
    """fp64 restatement of coda.py:43 (row / max(row sum, 1e-6)), 46-63 (base pseudo-counts) and 196 (multiplier) on
    the fixed-point sums; ``rest``: the compact slab's per-row term carried by every column."""
    C = conf_fx.shape[-1]
    v = conf_fx + (0 if rest is None else rest[..., None])
    conf = np.ldexp(v.astype(np.float64), -shift)
    conf = conf / np.maximum(conf.sum(-1, keepdims=True), 1e-6)
    if uniform:
        base = np.full((C, C), 2.0 / C)
    else:
        base = np.full((C, C), 1.0 / (C - 1) if off is None else off)
        np.fill_diagonal(base, 1.0)
    return multiplier * (base[None] + prior_strength * conf)


def prior_rtol(C):
    """k_init_dirichlets in fp32: the row sum (C / 32 terms per lane, a 5-level tree, non-negative terms) and the int64
    -> fp64 -> fp32 conversions, then conf / rs, prior_strength and the base rounded to fp32, the product, the sum of two
    non-negative terms and the multiplier: at most (ceil(C / 32) + 13) roundings of size u, relative."""
    return (math.ceil(C / 32) + 13) * U32


def contraction64(p, D):
    """coda.py:227-229 in fp64: U[n, c] = sum_h sum_s D[h, c, s] preds[h, n, s]."""
    return np.einsum("hns,hcs->nc", p.astype(np.float64), D.astype(np.float64))


def xi64(U):
    return U / np.maximum(U.sum(1, keepdims=True), 1e-12)


def fx_sum(xi32, shift):
    """sum_n rint(xi * 2^s) per column, int64: the fixed-point column sums of pi_hat_xi."""
    return np.rint(xi32.astype(np.float64) * 2.0 ** shift).astype(np.int64).sum(0)


# ------------------------------------------------------------------------------------------------------------------
# CPU tier: the models against the reference's own numbers
# ------------------------------------------------------------------------------------------------------------------
def _ctor(g):
    c = g["ctor"]
    return 1 - c.get("alpha", 0.9), c.get("multiplier", 2.0), bool(c.get("disable_diag_prior", False))


@pytest.mark.parametrize("name", golden_names())
def test_prior_and_contraction_models_reproduce_the_goldens(name):
    """The prior model on the integer confusion sums of the golden's slab gives the reference's initial dirichlets, and
    the fp64 contraction on them its initial pi_hat (and pi_hat_xi), at the oracle tests' tolerances -- each where the
    golden stores it (the H = 256 golden stores pi_hat only, cfg2 no pi_hat_xi)."""
    g = load_golden(name)
    preds, _ = golden_slab(g)
    p = preds.numpy()
    H, N, C = p.shape
    _, _, _, pseudo = scan_model(p)
    shift = fx_shift_of(N)
    ps, mult, uniform = _ctor(g)
    D = prior_model(confusion_model(p, pseudo, shift, C), shift, ps, mult, uniform)
    if "init_dirichlets" in g:
        _report("model", f"{name} init_dirichlets (rel)", float((np.abs(D - g["init_dirichlets"]) / g["init_dirichlets"]).max()), 2e-6)
        np.testing.assert_allclose(D, g["init_dirichlets"], rtol=2e-6, atol=1e-7)
    xi = xi64(contraction64(p, D))
    pi = xi.sum(0) / xi.sum()
    _report("model", f"{name} init_pi_hat (rel)", float((np.abs(pi - g["init_pi_hat"]) / g["init_pi_hat"]).max()), 2e-6)
    np.testing.assert_allclose(pi, g["init_pi_hat"], rtol=2e-6)
    if "init_pi_hat_xi" in g:
        np.testing.assert_allclose(xi, g["init_pi_hat_xi"], rtol=5e-6, atol=1e-9)


@pytest.mark.parametrize("name", ["traj_small_h32_n3000_c10", "traj_c100_h24_n400_c100", "traj_cfg2_h64_n50000_c10"])
def test_integer_confusion_model_matches_the_oracle(name):
    """The int64 fixed-point confusion sums, row-normalised, against the oracle's fp32 soft_confusion (coda.py:28-43)
    on the same pseudo labels: equal to fp32 noise."""
    g = load_golden(name)
    preds, _ = golden_slab(g)
    p = preds.numpy()
    C = p.shape[2]
    _, _, _, pseudo = scan_model(p)
    assert np.array_equal(pseudo, preds.mean(0).argmax(-1).numpy())          # the oracle's pseudo labels
    shift = fx_shift_of(p.shape[1])
    fx = np.ldexp(confusion_model(p, pseudo, shift, C).astype(np.float64), -shift)
    got = fx / np.maximum(fx.sum(-1, keepdims=True), 1e-6)
    ref = coda_oracle.soft_confusion(torch.from_numpy(pseudo), preds).numpy()
    _report("model", f"{name} soft_confusion", float(np.abs(got - ref).max()), 1e-6)
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------
# GPU plumbing
# ------------------------------------------------------------------------------------------------------------------
def _nat():
    from coda_b200 import _native as nat
    return nat, nat.load()


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return None if t is None else t.data_ptr()


@contextlib.contextmanager
def _env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    for k, v in kw.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


DTYPES = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


def widen(t):
    """Host fp32 copy of a device slab: the exact widening every kernel reads."""
    return t.float().cpu().numpy()


def tie_slab(H, N, C, seed, dtype):
    """(H, N, C) post-softmax-like slab with arg-max ties built in: item n of the first 64 repeats its maximum at
    classes c, c + 1, c + 32 and c + 64 (one or several of them, same lane or different lanes); item 64 has two classes
    whose ensemble sums are equal (every value a multiple of 2^-6, so the fp32 sums are exact); for 16-bit slabs item
    65 holds two fp32 values that collide after rounding to the stored width."""
    rng = np.random.default_rng(seed)
    p = rng.uniform(0.0, 0.5, (H, N, C)).astype(np.float32)
    for n in range(min(64, N)):
        c = n % C
        peers = [x % C for x in (c, c + 1, c + 32, c + 64)][: 1 + n % 4]
        for h in range(H):
            p[h, n, peers] = np.float32(0.75)
    if N > 64 and C >= 3:
        p[:, 64] = np.float32(2.0 ** -6)
        p[0, 64, 1] = p[1 % H, 64, 2] = np.float32(0.5)
        if H == 1:
            p[0, 64, 2] = np.float32(0.5)
    if N > 65 and dtype != torch.float32:
        p[:, 65, C - 1] = np.float32(0.8)
        p[:, 65, 0] = np.float32(0.8) + np.float32(1e-5)                 # the same value in bf16 and in fp16
    return torch.from_numpy(p).to(dtype).cuda()


# ------------------------------------------------------------------------------------------------------------------
# scan
# ------------------------------------------------------------------------------------------------------------------
def launch_scan(preds, fmt, H, N, C):
    nat, lib = _nat()
    dev = preds.device
    hard = torch.full((N, H), POISON & 0x7FFF, dtype=torch.int16, device=dev)
    pseudo = torch.full((N,), POISON, dtype=torch.int32, device=dev)
    dis = torch.full((N,), 0xA5, dtype=torch.uint8, device=dev)
    E = torch.full((N, C), NAN, device=dev)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    nat.check(lib.coda_b200_scan_slab_x(_p(preds), fmt, N * C, H, N, C, _p(hard), _p(pseudo), _p(dis), _p(E), _p(flags),
                                        _s()), "scan_slab_x")
    torch.cuda.synchronize()
    return (hard.cpu().numpy().astype(np.int64) & 0xFFFF, dis.cpu().numpy(), E.cpu().numpy(), pseudo.cpu().numpy(),
            int(flags.item()))


def scan_path(esz, H, N, C, ptr):
    """The selection rule of scan_slab: bulk-TMA kernel (template KC = ceil(C / 32)) when C <= 128, every copy is whole
    16-byte units and its 4-stage ring fits 200 KB of shared memory; else the generic kernel."""
    e16 = 16 // esz
    smem = 4 * ((32 * C * esz + 127) // 128 * 128) + (32 * H * 2 + 15) // 16 * 16 + 32
    if (C <= 128 and (N * C) % e16 == 0 and (32 * C) % e16 == 0 and ((N % 32) * C) % e16 == 0 and ptr % 16 == 0
            and smem <= 200 * 1024):
        return f"tma KC={(C + 31) // 32}"
    return "generic"


SCAN_CASES = [(7, 301, 5, "f32", "generic"), (7, 300, 100, "f32", "tma KC=4"), (7, 304, 100, "f16", "tma KC=4"),
              (7, 304, 100, "bf16", "tma KC=4"), (1, 96, 64, "f32", "tma KC=2"), (5, 300, 80, "f32", "tma KC=3"),
              (5, 304, 96, "bf16", "tma KC=3"), (9, 288, 20, "f32", "tma KC=1"), (7, 301, 150, "f32", "generic"),
              (7, 300, 150, "bf16", "generic"), (33, 97, 300, "f16", "generic")]


@pytest.mark.gpu
@pytest.mark.parametrize("H,N,C,dt,want", SCAN_CASES)
def test_scan_matches_host_model(H, N, C, dt, want):
    """hard / disagree / E / pseudo bit for bit against the host model on the widened slab, on purpose-built ties."""
    nat, _ = _nat()
    preds = tie_slab(H, N, C, seed=H * 7 + C, dtype=DTYPES[dt])
    hard, dis, E, pseudo, flags = launch_scan(preds, nat.slab_format(preds.dtype), H, N, C)
    path = scan_path(preds.element_size(), H, N, C, preds.data_ptr())
    assert path == want
    p = widen(preds)
    mh, md, mE, mp = scan_model(p)
    assert flags == 0
    assert np.array_equal(hard, mh), (path, np.argwhere(hard != mh)[:5])
    assert np.array_equal(dis.astype(bool), md) and set(np.unique(dis)) <= {0, 1}
    assert np.array_equal(E.view(np.int32), mE.view(np.int32)), path
    assert np.array_equal(pseudo, mp), (path, np.flatnonzero(pseudo != mp)[:5])
    _report("scan", f"H={H} N={N} C={C} {dt} {path} (mismatches)", 0.0, 0.0)
    lh, _, _, lp = scan_model(p, first=False)                  # negative control: last index among equal maxima
    assert not np.array_equal(hard, lh) and (C < 3 or N <= 64 or not np.array_equal(pseudo, lp))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [20, 150])
def test_scan_flags_out_of_range_and_non_finite_input(C):
    """NaN sets the non-finite bit only, < 0 and > 1.0001 the range bit; 1.0001 itself and 0 set nothing."""
    nat, _ = _nat()
    H, N = 3, 64
    base = torch.full((H, N, C), 1.0 / C)
    for val, want in ((1.0001, 0), (0.0, 0), (NAN, nat.FLAG_NONFINITE_INPUT), (-1e-30, nat.FLAG_RANGE_INPUT),
                      (1.0002, nat.FLAG_RANGE_INPUT), (float("inf"), nat.FLAG_NONFINITE_INPUT | nat.FLAG_RANGE_INPUT)):
        p = base.clone()
        p[2, N - 1, C - 1] = val
        flags = launch_scan(p.cuda(), nat.SLAB_F32, H, N, C)[4]
        assert flags == want, (val, hex(flags))


# ------------------------------------------------------------------------------------------------------------------
# confusion sums
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shift", [8, 30, 40])
@pytest.mark.parametrize("C", [5, 100, 128, 150, 300])
def test_confusion_sums_are_exact(C, shift):
    """Both kernels (class-sorted for C <= 128; shared-memory table up to C = 143, global atomics above) against
    the int64 host model, bit for bit, on an N-range view (items [40, 40 + N) of a longer slab).  The outputs
    accumulate, so they start at zero.  One class has no pseudo label."""
    nat, lib = _nat()
    H, Nall, N, lo = 5, 700, 613, 40
    rng = np.random.default_rng(C + shift)
    full = torch.from_numpy(rng.dirichlet(np.full(C, 0.3), (H, Nall)).astype(np.float32)).cuda()
    view = full[:, lo:lo + N]
    pseudo_np = rng.integers(1, C, N).astype(np.int32)                        # class 0 never
    pseudo = torch.from_numpy(pseudo_np).cuda()
    model = confusion_model(widen(view), pseudo_np, shift, C)
    kernels = (["sorted"] if C <= 128 else []) + ["accum"]
    for k in kernels:
        out = torch.zeros((H, C, C), dtype=torch.int64, device="cuda")
        if k == "sorted":
            order = torch.argsort(pseudo).to(torch.int32)
            nat.check(lib.coda_b200_confusion_sorted(_p(view), Nall * C, _p(pseudo), _p(order), H, N, C, shift, _p(out),
                                                     _s()), k)
        else:
            nat.check(lib.coda_b200_confusion_accum(_p(view), Nall * C, _p(pseudo), H, N, C, shift, _p(out), _s()), k)
        got = out.cpu().numpy()
        path = k if k == "sorted" else ("smem table" if C * C * 8 <= 160 * 1024 else "global atomics")
        _report("confusion", f"C={C} shift={shift} {path} (max |diff|)", float(np.abs(got - model).max()), 0.0)
        assert np.array_equal(got, model), (k, C, shift)
        assert not got[:, 0].any()
    floor = confusion_model(widen(view), pseudo_np, shift, C, rnd=np.floor)      # negative control: truncation
    assert not np.array_equal(got, floor)


# ------------------------------------------------------------------------------------------------------------------
# prior
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("uniform", [False, True])
@pytest.mark.parametrize("C,rest", [(6, False), (100, False), (300, False), (40, True)])
def test_init_dirichlets_matches_fp64(C, rest, uniform):
    """D against the fp64 prior on the same int64 sums, within prior_rtol(C) relative.  Row (h=0, c=1) is empty (the
    1e-6 clamp); ``rest``: the compact slab's per-row term."""
    nat, lib = _nat()
    H, shift, ps, mult = 4, 30, 0.1, 2.0
    rng = np.random.default_rng(C)
    fx = rng.integers(0, 2 ** shift, (H, C, C)).astype(np.int64) * rng.integers(0, 2, (H, C, C))
    fx[0, 1] = 0
    rs = rng.integers(0, 2 ** 20, (H, C)).astype(np.int64) if rest else None
    if rest:
        rs[0, 1] = 0
    D = torch.full((H, C, C), NAN, device="cuda")
    conf = torch.from_numpy(fx).cuda()
    rt = torch.from_numpy(rs).cuda() if rest else None
    nat.check(lib.coda_b200_init_dirichlets(_p(conf), _p(rt), H, C, shift, ps, mult, int(uniform), _p(D), _s()), "init")
    got = D.cpu().numpy().astype(np.float64)
    model = prior_model(fx, shift, ps, mult, uniform, rs)
    rel = float((np.abs(got - model) / model).max())
    _report("prior", f"C={C} uniform={uniform} rest={rest} (rel)", rel, prior_rtol(C))
    assert rel <= prior_rtol(C)
    assert np.allclose(got[0, 1], model[0, 1], rtol=prior_rtol(C), atol=0)        # the clamped empty row: base only
    wrong = prior_model(fx, shift, ps, mult, uniform, rs, off=1.0 / C) if not uniform else \
        prior_model(fx, shift, ps * (1 + 1e-3), mult, uniform, rs)
    assert (np.abs(got - wrong) / wrong).max() > prior_rtol(C)                    # negative control


# ------------------------------------------------------------------------------------------------------------------
# normalise
# ------------------------------------------------------------------------------------------------------------------
def launch_reduce(U, shift, xi=True):
    nat, lib = _nat()
    N, C = U.shape
    xo = torch.full_like(U, NAN) if xi else None
    pis = torch.zeros(C, dtype=torch.int64, device=U.device)
    flags = torch.zeros(1, dtype=torch.int32, device=U.device)
    nat.check(lib.coda_b200_pi_reduce(_p(U), N, C, shift, _p(xo), _p(pis), _p(flags), _s()), "pi_reduce")
    torch.cuda.synchronize()
    return xo, pis.cpu().numpy(), int(flags.item())


@pytest.mark.gpu
@pytest.mark.parametrize("N,C", [(1000, 7), (333, 128), (517, 129), (64, 1000), (40, 4096)])
def test_pi_reduce_matches_fp64_and_its_column_sums_are_exact(N, C):
    """xi = u / max(sum u, 1e-12) within (C/32 + 7) u relative of fp64 (lane sums, 5-level tree, one correctly
    rounded quotient); pisum = sum_n rint(xi_out 2^s) bit for bit.  Rows 3 and N-2 are all zero (the clamp).  U is
    read, not written."""
    nat, _ = _nat()
    shift = fx_shift_of(N)
    rng = np.random.default_rng(N + C)
    u = (rng.uniform(0, 1, (N, C)) ** 3 * rng.uniform(0.01, 100, (N, 1))).astype(np.float32)
    u[3] = 0
    u[N - 2] = 0
    U = torch.from_numpy(u).cuda()
    xo, pis, flags = launch_reduce(U, shift)
    assert flags == 0 and np.array_equal(U.cpu().numpy().view(np.int32), u.view(np.int32))
    x = xo.cpu().numpy()
    m = xi64(u.astype(np.float64))
    tol = (C / 32 + 7) * U32
    rel = float((np.abs(x - m) / np.maximum(m, 1e-300)).max())
    _report("normalise", f"N={N} C={C} xi (rel)", rel, tol)
    assert rel <= tol and not x[3].any() and not x[N - 2].any()
    assert np.array_equal(pis, fx_sum(x, shift))
    assert not np.array_equal(pis, np.floor(x.astype(np.float64) * 2.0 ** shift).astype(np.int64).sum(0))
    u2 = u.copy()
    u2[5, 0] = np.inf
    assert launch_reduce(torch.from_numpy(u2).cuda(), shift, xi=False)[2] & nat.FLAG_NONFINITE_PI


# ------------------------------------------------------------------------------------------------------------------
# label + rank-1 refresh
# ------------------------------------------------------------------------------------------------------------------
def label_slab(H, N, C, seed, dtype):
    """Item 0 unanimous (class 3 % C), item 1 split evenly between classes 1 and 2 (a count tie between majority and
    dissent), other items: each model right (class n % C) with probability 0.6.  0.6 on the predicted class, the rest
    spread unevenly."""
    rng = np.random.default_rng(seed)
    hard = np.where(rng.random((N, H)) < 0.6, (np.arange(N) % C)[:, None], rng.integers(0, C, (N, H)))
    hard[0] = 3 % C
    hard[1] = np.where(np.arange(H) % 2 == 0, 1 % C, 2 % C)
    p = rng.uniform(0.5, 1.5, (H, N, C)).astype(np.float32)
    hi, ni = np.arange(H)[:, None], np.arange(N)[None, :]
    p[hi, ni, hard.T] = 0
    p *= np.float32(0.4) / p.sum(-1, keepdims=True)
    p[hi, ni, hard.T] = np.float32(0.6)
    return torch.from_numpy(p).to(dtype)


def _selector(preds, **env):
    import gc
    from coda_b200 import CODA, TensorDataset
    gc.collect()                                   # engines no test holds any more give their constant-bank slots back
    with _env(**env):
        sel = CODA(TensorDataset(preds.cuda(), None))
    torch.cuda.synchronize()
    return sel


def term_buffers(e, P64):
    """(ptr, bytes, element size, fp64 host values) of every buffer a gather-list term may point into.  The ensemble
    sums are replaced by their exact fp64 values: the decoded list must then equal sum_h preds[h, n, j_h] in fp64."""
    Eex = P64.sum(0)                                                      # (N, C)
    bufs = [(e.preds.data_ptr(), e.preds.numel() * e.esz, e.esz, P64.reshape(-1))]
    if e.ens is not None:
        bufs.append((e.ens.data_ptr(), e.ens.numel() * 4, 4, Eex.reshape(-1)))
    cs = e.shadow_cs

    def class_major(v):                                                   # (N, C) -> [C][cs]
        out = np.zeros((v.shape[1], cs))
        out[:, : v.shape[0]] = v.T
        return out.reshape(-1)
    if e.shadow is not None:
        host = e.shadow.float().cpu().numpy().astype(np.float64).reshape(e.shadow.shape[0], -1)
        if e.esz == 4 and e.ens_shadow is not None:
            host[e.n_shadow] = class_major(Eex)
        bufs.append((e.shadow.data_ptr(), e.shadow.numel() * e.esz, e.esz, host.reshape(-1)))
    if e.ens_shadow is not None and e.esz != 4:
        bufs.append((e.ens_shadow.data_ptr(), e.ens_shadow.numel() * 4, 4, class_major(Eex)))
    if e.ens_shadow is not None:                                          # the class-major slot is E, transposed
        assert np.array_equal(e.ens_shadow[:, : e.N].T.cpu().numpy().view(np.int32), e.ens.cpu().numpy().view(np.int32))
    return bufs


def decode_terms(e, P64):
    """-> hdr (nterms, t'), per-term (sign, values over the N items), from the raw gather list."""
    raw = e.terms.cpu().numpy()
    nt, tp = int(raw[0]), int(raw[1])
    rec = raw[2:2 + 4 * nt].view(np.dtype([("off", "<i8"), ("sg", "<f4"), ("str", "<i4")]))
    bufs = term_buffers(e, P64)
    from coda_b200 import _native as nat
    n = np.arange(e.N)
    out = []
    for k, r in enumerate(rec):
        ens_base = k == 0 and tp >= 0 and e.fmt != nat.SLAB_F32
        base, el = (e._ens_base(), 4) if ens_base else (e._slab_ptr(), e.esz)
        a0 = base + int(r["off"]) * el
        hit = [b for b in bufs if b[0] <= a0 < b[0] + b[1]]
        assert len(hit) == 1 and hit[0][2] == el and (a0 - hit[0][0]) % el == 0, (k, r)
        assert r["sg"] in (1.0, -1.0) and r["str"] in (1, e.C), (k, r)
        idx = (a0 - hit[0][0]) // el + n * int(r["str"])
        assert idx.max() < hit[0][1] // el
        out.append((float(r["sg"]), hit[0][3][idx]))
    return nt, tp, out


def check_label_and_refresh(e, idx, t, P64, p32, hard, label):
    """One add_label by hand: step_label, then pi_rank1, each checked on the exact state it received."""
    nat, lib = _nat()
    H, N, C = e.H, e.N, e.C
    with e._on():
        e.label_stage(idx, t)
        torch.cuda.synchronize()
        D0 = e.D.cpu().numpy()
        U0 = e.U.cpu().numpy()
        e.jvec.fill_(POISON)
        e.terms.fill_(POISON)
        e.pisum.fill_(POISON)
        e._call("coda_b200_step_label", e.st, e._x(), e._s())
        torch.cuda.synchronize()
        # ---- label: D, jvec, pisum, gather list
        j = hard[idx]
        assert np.array_equal(e.jvec.cpu().numpy(), j) and not e.pisum.any()
        D1 = e.D.cpu().numpy()
        want = D0.copy()
        want[np.arange(H), t, j] = D0[np.arange(H), t, j] + np.float32(e.lr)       # one fp32 add of lr
        assert np.array_equal(D1.view(np.int32), want.view(np.int32))
        cnt = np.bincount(j, minlength=C)
        tp, M = int(cnt.argmax()), H - int(cnt.max())                              # lowest of the most common classes
        short = e.ens is not None and 2 * M < H
        nt, hdr_tp, terms = decode_terms(e, P64)
        assert (nt, hdr_tp) == ((1 + 2 * M, tp) if short else (H, -1)), (label, idx, nt, hdr_tp, M, tp)
        S = sum(sg * v for sg, v in terms)
        direct = P64[np.arange(H), :, j].sum(0)                                    # sum_h preds[h, n, j_h]
        assert np.abs(S - direct).max() <= 1e-12 * H, (label, idx)
        # ---- rank-1 refresh on that state
        U = e.U
        ens = _p(e.ens) if e.fmt == nat.SLAB_F32 else e._ens_base()
        e._slab_call("coda_b200_pi_rank1", ens, H, N, C, _p(e.sel), e.lr, e.fx_shift, _p(e.terms), _p(U), _p(e.pisum),
                     _p(e.flags), 8, e.const_slot, e._s())
        torch.cuda.synchronize()
        assert int(e.flags.item()) == 0
        U1 = U.cpu().numpy()
        others = np.arange(C) != t
        assert np.array_equal(U1[:, others].view(np.int32), U0[:, others].view(np.int32))
        lr = float(np.float32(e.lr))
        # bound of the kernel's chain: fmaf over the terms in list order (u |partial sum| each), the shortcut's E
        # (an H-term fp32 sum of non-negative values: (H - 1) u E), lr * d, and the add into U
        vals = np.stack([sg * v for sg, v in terms])
        partial = np.abs(np.cumsum(vals, 0)).sum(0)
        Eterm = terms[0][1] if short else 0.0
        model = U0[:, t].astype(np.float64) + lr * direct
        bound = lr * (U32 * partial + (H - 1) * U32 * Eterm + U32 * np.abs(direct)) + U32 * np.abs(model)
        bound = 1.01 * bound + 1e-45
        err = np.abs(U1[:, t] - model)
        _report("rank-1", f"{label} item {idx} (err / bound)", float((err / bound).max()), 1.0)
        assert (err <= bound).all(), (label, idx, float((err / bound).max()))
        jw = j.copy()
        jw[0] = (jw[0] + 1) % C                                                    # negative control: one model's class
        wrong = U0[:, t].astype(np.float64) + lr * P64[np.arange(H), :, jw].sum(0)
        assert (np.abs(U1[:, t] - wrong) > bound).any()
        # ---- the refreshed column sums are exactly what the full normalisation gives on the refreshed U
        _, pis, fl = launch_reduce(U, e.fx_shift, xi=False)
        assert fl == 0 and np.array_equal(e.pisum.cpu().numpy(), pis), label
        assert np.array_equal(U.cpu().numpy().view(np.int32), U1.view(np.int32))


R1_CASES = [
    # (H, N, C, dtype, env, expected path)
    (6, 300, 20, "f32", {}, dict(kc=1, const=True, shadow="all", ens="class-major")),
    (6, 300, 50, "f32", {"CODA_B200_R1_CONST": 0}, dict(kc=2, const=False, shadow="all", ens="class-major")),
    (6, 300, 100, "f16", {"CODA_B200_SHADOW_MODELS": 3}, dict(kc=4, const=True, shadow="some", ens="class-major")),
    (6, 300, 100, "bf16", {"CODA_B200_SHADOW": 0}, dict(kc=4, const=True, shadow="none", ens="item-major")),
    (6, 300, 100, "f32", {"CODA_B200_SHADOW": 0, "CODA_B200_ENS": 0}, dict(kc=4, const=True, shadow="none", ens="none")),
    (6, 300, 300, "f32", {"CODA_B200_SHADOW_MODELS": 2}, dict(kc=0, const=False, shadow="some", ens="class-major")),
    (7, 300, 300, "bf16", {"CODA_B200_ENS": 0}, dict(kc=0, const=False, shadow="all", ens="none")),
    (1, 200, 10, "f32", {}, dict(kc=1, const=True, shadow="all", ens="class-major")),
    (1024, 300, 12, "f32", {"CODA_B200_SHADOW_MODELS": 500}, dict(kc=1, const=True, shadow="some", ens="class-major")),
    (5, 257, 3300, "f32", {}, dict(kc=0, const=False, shadow="all", ens="class-major")),      # above the old 3200 - H/2
]


@pytest.mark.gpu
@pytest.mark.parametrize("H,N,C,dt,env,path", R1_CASES, ids=[f"H{c[0]}-C{c[2]}-{c[3]}-{i}" for i, c in enumerate(R1_CASES)])
def test_label_and_rank1_refresh_match_host_models(H, N, C, dt, env, path):
    """step_label and pi_rank1 on a unanimous item, a majority / dissent count tie and ordinary items.  N = 300 and
    200 are not multiples of the 32-item warp span or the 256-item CTA span."""
    preds = label_slab(H, N, C, seed=H + C, dtype=DTYPES[dt])
    sel = _selector(preds, **env)
    e = sel.engine
    try:
        kc = 1 if C <= 32 else 2 if C <= 64 else 4 if C <= 128 else 0
        slot_terms = (2 * H + 63) // 64 * 64                              # pi_rank1's constant-bank rule
        use_const = e.const_slot >= 0 and (e.const_slot + 1) * slot_terms <= 3584 and C <= 128
        assert kc == path["kc"] and use_const == path["const"], (e.const_slot, H)
        assert {0: "none", H: "all"}.get(e.n_shadow, "some") == path["shadow"]
        assert ("none" if e.ens is None else "class-major" if e.ens_shadow is not None else "item-major") == path["ens"]
        p32 = widen(preds)
        P64 = p32.astype(np.float64)
        hard = p32.argmax(-1).T
        for k, idx in enumerate([0, 1, 17, N - 1]):
            check_label_and_refresh(e, idx, (idx * 7 + k) % C, P64, p32, hard, f"H={H} C={C} {dt}")
    finally:
        sel.close()


# ------------------------------------------------------------------------------------------------------------------
# long run of the host-free loop
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_incremental_marginals_hold_over_a_long_run():
    """1 200 labels through run_steps, 90 % of them of class 0, so column 0 of U absorbs almost every rank-1 rounding.
    U against the fp64 contraction on the final D within: the initial SIMT pass (an H C-term FMA chain of non-negative
    terms, H C u relative) plus, for every update of the column, the rank-1 chain's bound (check_label_and_refresh,
    with the list's partial sums bounded by nterms times the sum of |terms|) and the fp32 rounding of the D entries
    the update moved.  pi_hat_xi follows from U; pisum is pi_reduce of U bit for bit."""
    from coda_b200.synth import synth
    H, N, C, K = 16, 3000, 10, 1200
    preds, _ = synth(H, N, C, seed=21)
    rng = np.random.default_rng(0)
    labels = torch.from_numpy(np.where(rng.random(N) < 0.9, 0, rng.integers(1, C, N))).to(torch.int64)
    sel = _selector(preds)
    e = sel.engine
    try:
        assert e._pi_tc is False and e.ens is not None
        sel.run_steps(K, labels)
        torch.cuda.synchronize()
        picks = np.asarray(sel.history()[0])[:K]
        assert len(set(picks.tolist())) == K
        p = preds.numpy().astype(np.float64)
        hard = preds.numpy().argmax(-1).T
        D = e.D.cpu().numpy()
        U = e.U.cpu().numpy()
        U64 = contraction64(preds.numpy(), D)
        lr = float(np.float32(e.lr))
        bound = H * C * U32 * U64
        ts = labels.numpy()[picks]
        Eex = p.sum(0)
        for idx, t in zip(picks, ts):
            j = hard[idx]
            cnt = np.bincount(j, minlength=C)
            tp, M = int(cnt.argmax()), H - int(cnt.max())
            pj = p[np.arange(H), :, j]                                        # (H, N)
            direct = pj.sum(0)
            if 2 * M < H:
                dis = j != tp
                A = Eex[:, tp] + (pj[dis] + p[np.flatnonzero(dis), :, tp]).sum(0)
                nt, Et = 1 + 2 * M, Eex[:, tp]
            else:
                A, nt, Et = direct, H, 0.0
            dD = U32 * (pj * D[np.arange(H), t, j][:, None]).sum(0)
            bound[:, t] += lr * (U32 * nt * A + (H - 1) * U32 * Et + U32 * direct) + U32 * U64[:, t] + dD
        bound *= 1.01
        err = np.abs(U - U64)
        col0 = int((ts == 0).sum())
        _report("long run", f"U, {K} labels ({col0} on column 0) (err / bound)", float((err / bound).max()), 1.0)
        _report("long run", "U column 0 (rel)", float((err[:, 0] / U64[:, 0]).max()), float((bound[:, 0] / U64[:, 0]).max()))
        assert col0 >= 0.8 * K and (err <= bound).all()
        xi = sel.pi_hat_xi.cpu().numpy()
        x64 = xi64(U64)
        relU = bound / U64
        xb = x64 * (relU + relU.max(1, keepdims=True) + (C / 32 + 7) * U32) * 1.01
        xe = np.abs(xi - x64)
        _report("long run", "pi_hat_xi (rel)", float((xe / x64).max()), 5e-6)
        _report("long run", "pi_hat_xi (err / bound)", float((xe / xb).max()), 1.0)
        assert (xe <= xb).all()
        _, pis, fl = launch_reduce(e.U, e.fx_shift, xi=False)
        assert fl == 0 and np.array_equal(e.pisum.cpu().numpy(), pis)
    finally:
        sel.close()


# ------------------------------------------------------------------------------------------------------------------
# the documented class count
# ------------------------------------------------------------------------------------------------------------------
def _chunked_oracle_state(preds_dev, D_dev, chunk=64):
    """The oracle's dirichlets (coda.py:195-196: its soft_confusion and its base pseudo-counts), compared chunk by chunk
    of models with the engine's D on the device (rtol 3e-6, atol 1e-7), and its consensus marginals (coda.py:226-233)
    on that D, accumulated over the same chunks: two (H, C, C) posteriors of H = 1024, C = 2700 do not fit at once."""
    H, N, C = preds_dev.shape
    pseudo = preds_dev.mean(0).argmax(-1)
    base = coda_oracle.dirichlet_prior(torch.zeros((1, C, C)), 0.0, False)[0].to(preds_dev.device)
    adj = torch.zeros((N, C), dtype=torch.float64, device=preds_dev.device)
    worst = 0.0
    for h0 in range(0, H, chunk):
        p = preds_dev[h0:h0 + chunk]
        Do = 2.0 * (base + 0.1 * coda_oracle.soft_confusion(pseudo, p))
        d = D_dev[h0:h0 + chunk]
        worst = max(worst, float(((d - Do).abs() - 3e-6 * Do.abs()).max()))
        adj += torch.einsum("hcs,hns->nc", d.double(), p.double())
        del Do
    xi = adj / adj.sum(-1, keepdim=True).clamp(min=1e-12)
    return worst, xi, xi.sum(0) / xi.sum()


@pytest.mark.gpu
@pytest.mark.parametrize("H,N,C", [(3, 48, 3201), (3, 40, 4096), (128, 40, 3150)])
def test_documented_class_count_follows_the_oracle(H, N, C):
    """C up to 4096 and H up to 1024 (engine.py, DESIGN §9): construction, get_next_item_to_label and add_label at
    class counts whose per-warp column sums overflowed shared memory (pi_reduce above C = 3200, the generic rank-1 row
    pass above C = 3200 - H/2) and whose mixture staging exceeded the default 48 KB (C >= 4086), and where a plain
    fp32 chain of the full pass drifts from the oracle by 1e-4.  Small H: the full oracle (dirichlets, pi_hat,
    pi_hat_xi, P(best), EIG on the candidates, the posterior after three labels).  H = 128: the oracle's prior and
    marginals by chunks of models on the device, and P(best) from its quadrature, class by class.  H = 128,
    C = 3150 lies above the old rank-1 limit 3200 - H/2."""
    import random
    from coda_b200.synth import synth
    preds, labels = synth(H, N, C, seed=C)
    small = H <= 8
    sel = _selector(preds)
    e = sel.engine
    try:
        if small:
            random.seed(0)
            ora = coda_oracle.OracleSelector(preds)
            np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), ora.dirichlets.numpy(), rtol=3e-6, atol=1e-7)
        for step in range(3):
            if small:
                # the oracle's marginals evaluated in fp64: its fp32 einsum over 4096 classes is itself ~5e-6 off
                xi64o, pi64o = coda_oracle.consensus_marginals(ora.dirichlets.double(), preds.double())
                rel = float(((sel.pi_hat.cpu().double() - pi64o).abs() / pi64o).max())
                rel32 = float(((sel.pi_hat.cpu() - ora.pi_hat).abs() / ora.pi_hat).max())
                _report("C=4096", f"H={H} C={C} step {step} pi_hat (rel; fp32 oracle {rel32:.1e})", rel, 5e-6)
                np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), pi64o.numpy(), rtol=5e-6, atol=1e-9)
                np.testing.assert_allclose(sel.pi_hat_xi.cpu().numpy(), xi64o.numpy(), rtol=5e-6, atol=1e-9)
                np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), ora.get_pbest().numpy(), atol=1e-5)
                i_ref, q_ref = ora.get_next_item_to_label()
                i, q = sel.get_next_item_to_label()
                np.testing.assert_allclose(e.eig.cpu().numpy()[np.asarray(ora.last_cand)], ora.last_q.numpy(), atol=5e-6)
                ora.add_label(i_ref, int(labels[i_ref]), q_ref)
            else:
                pd = preds.cuda()
                worst, xi, pi = _chunked_oracle_state(pd, e.D)        # marginals on the engine's (checked) posterior
                assert step > 0 or worst <= 1e-7, worst
                rel = float(((sel.pi_hat.cuda().double() - pi).abs() / pi).max())
                _report("C=4096", f"H={H} C={C} step {step} pi_hat (rel)", rel, 5e-6)
                np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), pi.cpu().numpy(), rtol=5e-6, atol=1e-9)
                np.testing.assert_allclose(sel.pi_hat_xi.cpu().numpy(), xi.cpu().numpy(), rtol=5e-6, atol=1e-9)
                a = torch.diagonal(e.D, dim1=-2, dim2=-1)
                b = e.D.sum(-1) - a
                pb = torch.cat([coda_oracle.pbest_rows(a[:, c0:c0 + 300].T.contiguous(), b[:, c0:c0 + 300].T.contiguous())
                                for c0 in range(0, C, 300)])
                m0 = (pb * sel.pi_hat.cuda()[:, None]).sum(0, keepdim=True)
                np.testing.assert_allclose(sel.get_pbest().cpu().numpy(), m0.cpu().numpy(), atol=1e-5)
                del pd, pb, a, b
                i_ref, q = sel.get_next_item_to_label()
            sel.add_label(i_ref, int(labels[i_ref]), q)
            torch.cuda.synchronize()
        if small:
            np.testing.assert_allclose(sel.dirichlets.cpu().numpy(), ora.dirichlets.numpy(), rtol=3e-6, atol=1e-7)
            np.testing.assert_allclose(sel.pi_hat.cpu().numpy(), coda_oracle.consensus_marginals(
                ora.dirichlets.double(), preds.double())[1].numpy(), rtol=5e-6, atol=1e-9)
    finally:
        sel.close()
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------------------------
# compact slab: label + the two rank-1 refresh kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["index", "slab"])
@pytest.mark.parametrize("H,N,C,K", [(9, 300, 20, 3), (6, 257, 150, 4), (12, 300, 600, 2)])
def test_compact_rank1_refresh_matches_fp64(H, N, C, K, kernel):
    """pi_rank1_index (the inverted index; KCU = 4, 16, 32: the compact slab is built up to C = 1024) and pi_rank1_compact (the slab scan) on the state
    step_label left.  The gather list names (model, class): decoded on the densified slab it must give
    sum_h preds[h, n, j_h] in fp64.  Column t against U + lr sum_h preds[h, n, j_h] within the kernel's bound:
      slab   E[n][t'] (an H-term fp32 sum, (H - 1) u E) then an fmaf chain over the terms (u |partial sum| each);
      index  R[n] = sum_h rest_h (fp32, (H - 1) u R) plus the int64 sum of (p - rest) at 2^-40 (2^-41 per entry) and
             its conversion (u |delta|);
    then lr d and the add into U.  Every other column keeps its bits, pisum is pi_reduce of the refreshed U bit for bit,
    and the index path's per-item delta is back to zero."""
    from coda_b200 import CODA, CompactDataset, CompactSlab
    from coda_b200.synth import synth_compact
    import gc
    ids, probs, _ = synth_compact(H, N, C, K, seed=C + K)
    slab = CompactSlab(ids, probs, C)
    gc.collect()
    with _env(CODA_B200_COMPACT_INDEX=None if kernel == "index" else 0):
        sel = CODA(CompactDataset(slab.to("cuda")))
    torch.cuda.synchronize()
    e = sel.engine
    try:
        assert (e.cidx is not None) == (kernel == "index") and e.compact is not None and e.ens is not None
        P64 = slab.densify().numpy().astype(np.float64)
        pr = probs.numpy()
        s32 = pr[..., 0].copy()
        for j in range(1, K):
            s32 = s32 + pr[..., j]
        rest64 = ((np.float32(1) - s32) * np.float32(1.0 / (C - K))).astype(np.float64)      # (H, N)
        hard = e.hard.cpu().numpy().astype(np.int64) & 0xFFFF             # the engine's own p_h(n)
        lr = float(np.float32(e.lr))
        for k, idx in enumerate([0, 1, 17, N - 1]):
            t = (idx * 5 + k) % C
            with e._on():
                e.label_stage(idx, t)
                torch.cuda.synchronize()
                U0 = e.U.cpu().numpy()
                e.jvec.fill_(POISON)
                e.terms.fill_(POISON)
                e.pisum.fill_(POISON)
                e._call("coda_b200_step_label", e.st, e._x(), e._s())
                torch.cuda.synchronize()
                j = hard[idx]
                assert np.array_equal(e.jvec.cpu().numpy(), j) and not e.pisum.any()
                cnt = np.bincount(j, minlength=C)
                tp, M = int(cnt.argmax()), H - int(cnt.max())
                short = 2 * M < H
                raw = e.terms.cpu().numpy()
                nt, hdr_tp = int(raw[0]), int(raw[1])
                assert (nt, hdr_tp) == ((2 * M, tp) if short else (H, -1)), (nt, hdr_tp, M, tp)
                rec = raw[2:2 + 4 * nt].view(np.dtype([("off", "<i8"), ("sg", "<f4"), ("str", "<i4")]))
                direct = P64[np.arange(H), :, j].sum(0)
                vals = ([P64[:, :, tp].sum(0)] if short else []) + [float(r["sg"]) * P64[int(r["off"]), :, int(r["str"])]
                                                                    for r in rec]
                assert np.abs(sum(vals) - direct).max() <= 1e-12 * H
                if kernel == "index":
                    ix = e.cidx
                    e._call("coda_b200_pi_rank1_index", _p(ix["off"]), _p(ix["ent"]), _p(ix["rest"]), _p(e.jvec), H, N, C,
                            _p(e.sel), e.lr, e.fx_shift, _p(e.terms), _p(ix["delta"]), _p(e.U), _p(e.pisum), _p(e.flags),
                            e._s(), n=2)
                else:
                    e._call("coda_b200_pi_rank1_compact", _p(e.compact.ids), _p(e.compact.probs), e.model_stride,
                            _p(e.ens), H, N, C, K, _p(e.sel), e.lr, e.fx_shift, _p(e.terms), _p(e.U), _p(e.pisum),
                            _p(e.flags), e._s())
                torch.cuda.synchronize()
                assert int(e.flags.item()) == 0
                U1 = e.U.cpu().numpy()
                others = np.arange(C) != t
                assert np.array_equal(U1[:, others].view(np.int32), U0[:, others].view(np.int32))
                model = U0[:, t].astype(np.float64) + lr * direct
                if kernel == "index":
                    R = rest64.sum(0)
                    delta = direct - R
                    chain = (H - 1) * U32 * R + H * 2.0 ** -41 + U32 * np.abs(delta)
                    assert not e.cidx["delta"].any()
                else:
                    E = P64[:, :, tp].sum(0) if short else 0.0
                    partial = np.abs(np.cumsum(np.stack(vals), 0)).sum(0) - (np.abs(vals[0]) if short else 0.0)
                    chain = U32 * partial + (H - 1) * U32 * E
                bound = 1.01 * (lr * (chain + U32 * np.abs(direct)) + U32 * np.abs(model)) + 1e-45
                err = np.abs(U1[:, t] - model)
                _report("rank-1", f"compact {kernel} H={H} C={C} K={K} item {idx} (err / bound)", float((err / bound).max()), 1.0)
                assert (err <= bound).all()
                jw = j.copy()
                jw[0] = (jw[0] + 1) % C
                assert (np.abs(U1[:, t] - (U0[:, t] + lr * P64[np.arange(H), :, jw].sum(0))) > bound).any()
                _, pis, fl = launch_reduce(e.U, e.fx_shift, xi=False)
                assert fl == 0 and np.array_equal(e.pisum.cpu().numpy(), pis)
    finally:
        sel.close()
