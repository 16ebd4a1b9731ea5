"""Golden fixtures for the epsilon search's metrics and selection, made by RUNNING THE REFERENCE SCRIPT's own
``run_grid_search`` (scripts/modelselector/modelselector_eps_gridsearch_v2.py) on scripted runs.

    CODA_REFERENCE_PATH=<reference checkout> python tests/golden/make_eps_search_golden.py

Only the ModelPicker runs are scripted: ``run_realisation`` returns a given best model per step, with the pool's
accuracies from the script's own ``calculate_model_ranking`` on given hard predictions and oracle labels; the loader,
the majority vote and the realisations are replaced by stand-ins for the same reason.  Everything after that (success,
accuracy, smoothing, fastest_t, best_avg / best_fast) is the script's code.  -> tests/golden/eps_search_<case>.npz:
inputs ``best`` [E][R][B], ``pool_acc`` [R][H] (integer counts), ``pool_size``, ``epsilons``, ``threshold``; outputs
``success_mean`` / ``acc_mean`` [E][B], ``avg_success`` / ``fastest_t`` [E], ``best_avg``, ``best_fast``.
"""
import argparse
import importlib.util
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("CODA_REFERENCE_PATH", "")


def load_script():
    for k in [k for k in sys.modules if k == "coda" or k.startswith("coda.")]:
        del sys.modules[k]
    sys.path.insert(0, REF)
    for name in ("matplotlib", "matplotlib.pyplot"):
        sys.modules.setdefault(name, types.ModuleType(name))
    path = os.path.join(REF, "scripts", "modelselector", "modelselector_eps_gridsearch_v2.py")
    spec = importlib.util.spec_from_file_location("ref_eps_gridsearch", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.tqdm = lambda it, *a, **k: it
    return mod


def crafted(rng):
    """E = 5: e0 always picks a top model, e1 the same runs (ties with e0 in both selections), e2 never (no t reaches
    the threshold), e3 only at t = 5 (reached there, but the smoothed value fails), e4 a random mix."""
    R, P, H, C, B = 6, 20, 5, 4, 12
    oracle = rng.integers(0, C, (R, P))
    hard = rng.integers(0, C, (R, P, H))
    hard[:, :, 4] = (oracle + 1) % C                     # model 4 is never right: never a top model
    hard[:, :8, 0] = oracle[:, :8]                       # model 0 is usually top
    best = np.zeros((5, R, B), dtype=np.int64)
    for r in range(R):
        acc = (hard[r] == oracle[r][:, None]).sum(0)
        top = int(np.argmax(acc))
        best[0, r] = top
        best[1, r] = top
        best[2, r] = 4
        best[3, r] = 4
        best[3, r, 5] = top
        best[4, r] = rng.integers(0, H, B)
    return hard, oracle, best, [0.35, 0.4, 0.45, 0.46, 0.49], 0.9


def randomised(rng):
    R, P, H, C, B = 30, 50, 8, 3, 40
    oracle = rng.integers(0, C, (R, P))
    hard = np.where(rng.random((R, P, H)) < np.linspace(0.4, 0.95, H), oracle[:, :, None], rng.integers(0, C, (R, P, H)))
    E = 4
    best = np.zeros((E, R, B), dtype=np.int64)
    for e in range(E):                                   # mostly the accurate model from step 8 + 6 e on
        p = np.where(np.arange(B) >= 8 + 6 * e, 0.9, 0.15)
        best[e] = np.where(rng.random((R, B)) < p, H - 1, rng.integers(0, H, (R, B)))
    return hard, oracle, best, [0.36, 0.41, 0.46, 0.48], 0.5


def run_case(mod, hard, oracle, best, eps, threshold):
    R, P, H = hard.shape
    B = best.shape[2]
    calls = {"n": 0}

    def run_realisation(preds_hnc, subset_oracle, epsilon, budget, seed):
        e, r = calls["n"] // R, seed
        calls["n"] += 1
        assert budget == B and epsilon == eps[e] and np.array_equal(subset_oracle, oracle[r])
        return [int(b) for b in best[e, r]], mod.calculate_model_ranking(hard[r], subset_oracle)

    class Preds:                                         # what run_grid_search reads of the slab: its shape
        shape = (H, R * P, 2)

        def __getitem__(self, key):
            return None

    mod.Dataset = lambda path, device: types.SimpleNamespace(preds=Preds())
    mod.majority_vote_labels = lambda preds: oracle.reshape(-1)
    mod.create_realisations = lambda n, num_reals, pool_size: np.arange(R * P).reshape(R, P)
    mod.run_realisation = run_realisation
    args = argparse.Namespace(pool_size=P, budget=B, iterations=R, threshold=threshold,
                              epsilons=",".join(repr(e) for e in eps))
    res = mod.run_grid_search("scripted", args)
    m = [res["metrics"][e] for e in eps]
    pool_acc = np.stack([(hard[r] == oracle[r][:, None]).sum(0) for r in range(R)])
    return dict(best=best, pool_acc=pool_acc, pool_size=P, epsilons=np.array(eps), threshold=threshold,
                success_mean=np.array([x["success_mean"] for x in m]), acc_mean=np.array([x["acc_mean"] for x in m]),
                avg_success=np.array([x["avg_success"] for x in m]),
                fastest_t=np.array([float(x["fastest_t"]) for x in m]),
                best_avg=res["best_avg"], best_fast=res["best_fast"])


def main():
    mod = load_script()
    for name, make, seed in (("crafted", crafted, 1), ("random", randomised, 2)):
        out = run_case(mod, *make(np.random.default_rng(seed)))
        np.savez(os.path.join(HERE, f"eps_search_{name}.npz"), **out)
        print(name, out["best_avg"], out["best_fast"], out["fastest_t"], out["avg_success"])


if __name__ == "__main__":
    main()
