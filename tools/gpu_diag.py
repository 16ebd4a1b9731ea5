"""Stage-by-stage comparison of the CUDA path with the CPU oracle on one golden case (prints, never asserts).
    python tools/gpu_diag.py [golden name] > diag.txt
"""
import os
import random
import sys
import time
import traceback

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from helpers import coda_oracle, golden_slab, load_golden  # noqa: E402

from coda_b200 import CODA, TensorDataset  # noqa: E402


def err(name, a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    d = np.abs(a - b)
    rel = d / np.maximum(np.abs(b), 1e-30)
    print(f"  {name:28s} max_abs={d.max():.3e} max_rel={rel.max():.3e} (shape {a.shape})")


def main(name, mode):
    print("=" * 100, "\ncase", name, "mode", mode)
    g = load_golden(name)
    preds, labels = golden_slab(g)
    random.seed(0)
    ora = coda_oracle.OracleSelector(preds, **g["ctor"])
    dev = torch.device("cuda:0")
    t0 = time.time()
    random.seed(0)
    sel = CODA(TensorDataset(preds.to(dev), labels.to(dev)), mode=mode, **g["ctor"])
    torch.cuda.synchronize()
    print(f"construct {time.time()-t0:.3f}s  npairs={sel.engine.npairs} heavy={sel.engine.n_heavy} entries={sel.engine.n_entries} tiles={sel.engine.ntiles}")
    eng = sel.engine
    hard = eng.hard.cpu().numpy().astype(np.int64) & 0xFFFF
    print("  hard mismatch:", int((hard != ora.hard.T.numpy()).sum()), " disagree mismatch:",
          int((eng.disagree.cpu().numpy().astype(bool) != coda_oracle.disagreement_mask(ora.hard).numpy()).sum()))
    err("dirichlets vs golden", sel.dirichlets.cpu().numpy(), g["init_dirichlets"])
    err("pi_hat vs golden", sel.pi_hat.cpu().numpy(), g["init_pi_hat"])
    err("pi_hat_xi vs golden", sel.pi_hat_xi.cpu().numpy(), g["init_pi_hat_xi"])
    err("PB vs oracle", eng.PB[:, :eng.H].cpu().numpy(), ora.pbest_before().numpy())
    b0 = sel.get_best_model_prediction(); ora.get_best_model_prediction()
    print("  best model", int(b0), "golden", int(g["init_best_model"]))
    err("pbest vs golden", sel.get_pbest().cpu().numpy(), g["init_pbest"])
    for k in range(int(g["steps"])):
        t0 = time.time()
        idx, q = sel.get_next_item_to_label()
        dt = time.time() - t0
        ref = g["eig"][k]
        cand = ~np.isnan(ref)
        mine = eng.eig.cpu().numpy()
        rep = sel.last_report
        print(f" step {k}: idx={idx} (golden {int(g['idx'][k])}) q={q:.7f} (golden {float(g['q'][k]):.7f}) ties={rep['n_ties']} "
              f"ncand={rep['n_cand']} (golden {int(g['n_cand'][k])}) ref_eig[idx]-max={ref[idx]-np.nanmax(ref):.2e} t={dt*1e3:.1f}ms")
        err("eig vs golden", mine[cand], ref[cand])
        gidx = int(g["idx"][k])          # teacher forcing
        t = int(labels[gidx])
        sel.add_label(gidx, t, q)
        sel.get_best_model_prediction()
        err("pbest vs golden", sel.get_pbest().cpu().numpy()[0], g["pbest"][k])
        err("pi_hat vs golden", sel.pi_hat.cpu().numpy(), g["pi_hat"][k])
        err("dir row vs golden", sel.dirichlets[:, t].cpu().numpy(), g["dir_row"][k])
        err("xi head vs golden", sel.pi_hat_xi[:64].cpu().numpy(), g["xi_head"][k])
    print("  flags", int(eng.flags.item()), "launches", eng.counters)


if __name__ == "__main__":
    names = sys.argv[1:] or ["traj_tiny_h8_n300_c5", "traj_small_h32_n3000_c10", "traj_c100_h24_n400_c100",
                             "traj_dense_h16_n500_c12", "traj_nodiag_h10_n400_c6"]
    for n in names:
        for mode in ("incremental", "recompute", "recompute_all"):
            try:
                main(n, mode)
            except Exception:
                traceback.print_exc(file=sys.stdout)
