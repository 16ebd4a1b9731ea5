"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list: python tools/launch_list.py launches.csv

Per-kernel totals over the capture, then one steady-state acquisition step (the launches between two consecutive
k_step_select launches near the end of the device-loop section) with each kernel's share of the step."""
import collections
import csv
import re
import sys


def short(name):
    name = re.sub(r"\(.*$", "", name)                 # drop the argument list
    return name.replace("<unnamed>::", "").strip()


def main():
    path = sys.argv[1]
    rows = []
    with open(path, newline="") as f:
        for r in csv.reader(f):
            if len(r) >= 15 and r[0].isdigit() and r[12] == "gpu__time_duration.sum":
                ns = float(r[14].replace(",", ""))
                if r[13] == "us":
                    ns *= 1e3
                elif r[13] == "ms":
                    ns *= 1e6
                rows.append((int(r[0]), short(r[4]), ns / 1e6))
    rows.sort()
    print(f"# {len(rows)} launches captured")
    tot = collections.OrderedDict()
    for _, k, ms in rows:
        c, t = tot.get(k, (0, 0.0))
        tot[k] = (c + 1, t + ms)
    print(f"\n{'kernel':44s} {'launches':>8s} {'total ms':>10s} {'avg ms':>10s}")
    for k, (c, t) in sorted(tot.items(), key=lambda x: -x[1][1]):
        print(f"{k:44s} {c:8d} {t:10.3f} {t / c:10.4f}")
    sel = [i for i, (_, k, _) in enumerate(rows) if k == "k_step_select"]
    if len(sel) >= 4:
        a, b = sel[len(sel) // 2], sel[len(sel) // 2 + 1]
        step = rows[a:b]
        total = sum(ms for _, _, ms in step)
        print(f"\n# one steady-state step (launches {rows[a][0]}..{rows[b - 1][0]}), total {total:.3f} ms:")
        for _, k, ms in step:
            print(f"  {k:42s} {ms:8.4f} ms  {100 * ms / total:5.1f} %")


if __name__ == "__main__":
    main()
