"""Build the C-ABI shared library (sm_90a only) in-tree: coda_b200/lib/libcoda_b200.so."""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libcoda_b200.so")
SOURCES = ["api.cu", "xchg.cu", "slab.cu", "tables.cu", "pairs.cu", "pairs_tc.cu", "pi_tc.cu", "gain.cu", "step.cu", "step_defer.cu", "compact.cu", "baselines.cu",
           "eps_search.cu", "sample.cu", "bl_ref.cu", "true_loss.cu", "compact_build.cu", "preload.cu",
           "host_stage.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else "nvcc"


def _digest() -> str:
    h = hashlib.sha256()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))] + [os.path.join(ROOT, "include", "coda_b200.h")]
    for p in files:
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode()); h.update(f.read())   # location-independent: the .so travels
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _fresh(stamp, dig):
    return os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig


def is_fresh() -> bool:
    """True when the in-tree library was built from exactly the current csrc/ + include/ + flags."""
    return _fresh(os.path.join(LIBDIR, "build.sha256"), _digest())


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.sha256")
    dig = _digest()
    if not force and _fresh(stamp, dig):
        return LIB
    # one builder at a time (several ranks may import concurrently); the library is replaced atomically
    import fcntl
    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and _fresh(stamp, dig):
            return LIB
        return _build_locked(stamp, dig, verbose)


def _build_locked(stamp, dig, verbose):
    objs, log = [], []
    tmp_lib = LIB + f".tmp{os.getpid()}"
    for src in SOURCES:
        obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
        cmd = [_nvcc(), *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
        if r.returncode != 0:
            sys.stderr.write(log[-1])
            raise RuntimeError(f"nvcc failed on {src}")
        objs.append(obj)
    cmd = [_nvcc(), "-shared", "-o", tmp_lib, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
    if r.returncode != 0:
        sys.stderr.write(log[-1])
        raise RuntimeError("link failed")
    os.replace(tmp_lib, LIB)
    with open(os.path.join(LIBDIR, "build.log"), "w") as f:
        f.write("\n".join(log))
    with open(stamp, "w") as f:
        f.write(dig)
    if verbose:
        print("\n".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
