"""Per-kernel counts of the SASS mnemonics that prove wgmma / bulk-TMA use:
    python tools/sass_summary.py
"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "coda_b200", "lib", "libcoda_b200.so")
PAT = ["HGMMA", "WARPGROUP", "UBLKCP", "UTMALDG", "SYNCS", "LDGSTS", "MUFU.LG2", "MUFU.EX2", "HMMA", "REDUX", "ATOMG", "RED."]


def main():
    out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    cur, counts, sizes = None, collections.OrderedDict(), {}
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            raw = m.group(1)
            cur = subprocess.run(["c++filt", raw], capture_output=True, text=True).stdout.strip()
            cur = cur.replace("(anonymous namespace)::", "").split("(")[0]
            if cur.startswith("_Z"):                      # c++filt does not know nvcc's internal-linkage prefix
                mm = re.search(r"\d+(k_[a-z0-9_]+?)E", raw)
                cur = mm.group(1) if mm else raw
            counts.setdefault(cur, collections.Counter())
            sizes.setdefault(cur, 0)
            continue
        if cur and re.match(r"\s+/\*[0-9a-f]{4}\*/", line):
            sizes[cur] += 1
            for p in PAT:
                if p in line:
                    counts[cur][p] += 1
    print(f"# cuobjdump -sass {os.path.relpath(LIB, ROOT)} (sm_90a): instruction counts per kernel")
    print("# HGMMA = wgmma.mma_async, WARPGROUP = wgmma fence / arrive, UBLKCP = cp.async.bulk (1-D TMA),")
    print("# SYNCS = mbarrier ops, MUFU.LG2/EX2 = the entropy / exp terms")
    print(f"{'kernel':70s} {'instr':>7s}  " + "  ".join(f"{p:>8s}" for p in PAT))
    for k, c in counts.items():
        if "k_" not in k:
            continue
        print(f"{k[:70]:70s} {sizes[k]:7d}  " + "  ".join(f"{c.get(p, 0):8d}" for p in PAT))


if __name__ == "__main__":
    main()
