"""CPU side of the compact slab above C = 1024 (tests/test_compact_large_c.py runs the kernels): the NumPy model of the
compact scan, anchored to CompactSlab.densify(), and the C ABI surface of the compact path."""
import os
import re

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def scan_model(ids, probs, C, ascending=True):
    """coda_b200_scan_compact in NumPy fp32: rest = (1 - sum_j p_j) fp32(1 / (C - K)) (left-to-right sum), then per
    model h in ascending order row[id_j] += p_j - rest and rsum += rest; ens = row + rsum, pseudo = the first arg-max of
    ens / H.  Returns hard (N, H), disagree (N,), ens (N, C) fp32, pseudo (N,).  ``ascending=False`` adds the models in
    descending order: a wrong model that the kernels must not match."""
    ids = np.asarray(ids).astype(np.int64) & 0xFFFF
    probs = np.asarray(probs, dtype=np.float32)
    H, N, K = ids.shape
    s = probs[..., 0].copy()
    for j in range(1, K):
        s = (s + probs[..., j]).astype(np.float32)
    rest = ((np.float32(1) - s) * (np.float32(1) / np.float32(C - K))).astype(np.float32)     # (H, N)
    row = np.zeros((N, C), np.float32)
    rsum = np.zeros(N, np.float32)
    n = np.arange(N)
    for h in (range(H) if ascending else range(H - 1, -1, -1)):
        rsum = (rsum + rest[h]).astype(np.float32)
        for j in range(K):
            c = ids[h, :, j]
            ok = c < C
            row[n[ok], c[ok]] = (row[n[ok], c[ok]] + (probs[h, ok, j] - rest[h, ok]).astype(np.float32)).astype(np.float32)
    ens = (row + rsum[:, None]).astype(np.float32)
    pseudo = (ens / np.float32(H)).argmax(1).astype(np.int32)
    hard = ids[:, :, 0].T
    return hard, (hard != hard[:, :1]).any(1).astype(np.uint8), ens, pseudo


def _crafted(H, N, C, K, seed):
    rng = np.random.default_rng(seed)
    base = rng.integers(0, C, (H, N, 1))
    stride = rng.integers(1, max(2, C // K), (H, N, 1))
    ids = (base + stride * np.arange(K)) % C
    p = -np.sort(-rng.dirichlet(np.ones(K + 1), (H, N)).astype(np.float32)[..., :K], axis=-1)
    ids[:, 0] = (5 + 7 * np.arange(K)) % C                     # item 0: every model's top class is 5 (unanimous)
    return ids, p.astype(np.float32)


def test_scan_model_is_the_sum_of_the_densified_slab():
    """The model's ensemble row is sum_h densify()[h, n] up to the fp32 roundings of its two chains (H adds of rest,
    H K adds of p - rest into the row, then one add): within (H (K + 1) + 2) u (sum_h |densify| + 2 sum_h |rest|).  hard is densify's
    arg-max per model, pseudo the arg-max of the fp64 sum wherever it is not within that bound of a tie, and the
    descending-order model differs from it in some bit."""
    from coda_b200 import CompactSlab
    for H, N, C, K in [(33, 40, 1600, 4), (64, 25, 4096, 8), (7, 30, 3001, 1), (12, 20, 2048, 3)]:
        ids, p = _crafted(H, N, C, K, C + K)
        slab = CompactSlab(torch.from_numpy(ids.astype(np.int16)), torch.from_numpy(p), C)
        dense = slab.densify().numpy().astype(np.float64)
        hard, dis, ens, pseudo = scan_model(ids, p, C)
        want = dense.sum(0)
        rest_all = np.abs(dense.min(-1)).sum(0)[:, None]                # sum_h |rest_h|: both chains carry it for every h
        bound = (H * (K + 1) + 2) * 2.0 ** -24 * (np.abs(dense).sum(0) + 2 * rest_all) + 1e-30
        assert (np.abs(ens - want) <= bound).all(), (H, C, K)
        assert np.array_equal(hard, dense.argmax(-1).T) and dis[0] == 0
        srt = np.sort(want, axis=1)
        clear = (srt[:, -1] - srt[:, -2]) > 2 * bound.max(1)
        assert np.array_equal(pseudo[clear], want.argmax(1)[clear])
        assert not np.array_equal(scan_model(ids, p, C, ascending=False)[2].view(np.int32), ens.view(np.int32))


def test_scan_model_ties_go_to_the_first_class():
    H, C, K = 4, 2048, 2
    ids = np.tile(np.array([[C - 5, 3]]), (H, 1, 1))
    p = np.full((H, 1, K), 0.4, np.float32)
    _, _, ens, pseudo = scan_model(ids, p, C)
    assert ens[0, 3] == ens[0, C - 5] and pseudo[0] == 3


# the compact entries as the previous ABI (version 203) declared them: they keep their signatures
_COMPACT_ABI = {
    "coda_b200_scan_compact": "p p i64 i32 i64 i32 i32 p p p p p p",
    "coda_b200_confusion_compact": "p p i64 p i32 i64 i32 i32 i32 p p p",
    "coda_b200_pi_full_compact": "p p i64 p i32 i64 i32 i32 p p p p",
    "coda_b200_pi_rank1_compact": "p p i64 p i32 i64 i32 i32 p f64 i32 p p p p p",
    "coda_b200_compact_index_count": "p i64 i32 i64 i32 i32 p p",
    "coda_b200_compact_index_fill": "p p i64 i32 i64 i32 i32 p p p p",
    "coda_b200_pi_rank1_index": "p p p p i32 i64 i32 p f64 i32 p p p p p p",
}


def _code(t):
    import ctypes as ct
    return {ct.c_void_p: "p", ct.c_int64: "i64", ct.c_int32: "i32", ct.c_double: "f64", ct.c_int: "i32",
            ct.c_longlong: "i64", ct.c_float: "f32"}[t]


def test_the_abi_is_only_extended():
    """Every compact entry keeps its signature and the version stays 203; the one new entry,
    coda_b200_scan_compact_kernel, is scan_compact plus an int before the stream, and is declared in the header,
    bound in _native.py and exported by the library."""
    from coda_b200 import _native as nat
    assert nat.VERSION == 203
    hdr = open(os.path.join(ROOT, "include", "coda_b200.h")).read()
    assert re.search(r"#define CODA_B200_VERSION 203\b", hdr)
    declared = set(re.findall(r"\b(coda_b200_\w+)\s*\(", hdr))
    for name, sig in _COMPACT_ABI.items():
        assert name in declared
        assert " ".join(_code(a) for a in nat.SIGNATURES[name][1]) == sig, name
    new = "coda_b200_scan_compact_kernel"
    assert new in declared
    old = _COMPACT_ABI["coda_b200_scan_compact"].split()
    assert " ".join(_code(a) for a in nat.SIGNATURES[new][1]) == " ".join(old[:-1] + ["i32", "p"])
    lib = nat.load()
    assert getattr(lib, new).argtypes is not None
