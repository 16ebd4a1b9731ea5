"""CPU oracle for the CODA acquisition hot path.  TEST INFRASTRUCTURE ONLY.

This file is a CPU (torch fp32, ATen CPU kernels) restatement of the algorithm in
the reference's ``coda/coda.py`` -- the per-step expected-information-gain (EIG)
acquisition and the Bayesian posterior update.  It exists so that ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl
reference`` legs have something to check and time the CUDA path against.  The
product (``coda_b200``) never imports it; nothing here is a fallback.

Parity status: the reference ships no tests or golden vectors (SURVEY.md 8c), so
the oracle is pinned against *outputs of the reference itself*, run on CPU by
``tests/golden/make_golden.py`` and committed under
``tests/golden/``.  ``tests/test_oracle_golden.py`` replays them.

Every function cites the reference lines (the reference's ``coda/coda.py`` unless
another file is named) whose arithmetic it restates.  Arithmetic order follows the
reference where fp32 rounding is order-sensitive (the cumulative trapezoid, the
clamped leave-one-out product), so the oracle agrees with the reference to a few
fp32 ulps; the organisation (a flat state dict, row-major (rows, H) Beta batches,
no class hierarchy) is our own.
"""
from __future__ import annotations

import random as _pyrandom

import torch

QUAD_NODES = 256          # coda.py:79   num_points default
CDF_FLOOR = 1e-30         # coda.py:80   eps
EXP_CLAMP = 80.0          # coda.py:107  clamp(-80, 80)
ENT_FLOOR = 1e-12         # coda.py:254, 276
HYP_WEIGHT = 1.0          # coda.py:235  update_weight default
CHUNK = 100               # coda.py:235  chunk_size default


def _finite_or_raise(t: torch.Tensor, what: str) -> None:
    """coda/util.py:17-25 -- the reference raises RuntimeError('[NUMERIC ERROR] ...')."""
    if not bool(torch.isfinite(t).all()):
        bad = int((~torch.isfinite(t)).sum())
        raise RuntimeError(f"[NUMERIC ERROR] {what} has {bad} bad values (NaN/Inf) out of {t.numel()}")


def quad_grid(nodes: int = QUAD_NODES, device="cpu") -> torch.Tensor:
    """coda.py:86 -- the fp32 linspace grid (trap T1: not reproducible by a closed formula)."""
    return torch.linspace(1e-6, 1 - 1e-6, nodes, device=device)


def diag_beta_params(dirichlets: torch.Tensor):
    """coda.py:14-25 -- Beta(alpha, beta) of the diagonal of each Dirichlet row.
    dirichlets (..., H, C, C) -> alpha, beta (..., H, C)."""
    a = torch.diagonal(dirichlets, dim1=-2, dim2=-1)
    b = dirichlets.sum(dim=-1) - a
    return a, b


def soft_confusion(pseudo_labels: torch.Tensor, preds: torch.Tensor) -> torch.Tensor:
    """coda.py:28-43 (mode='soft') -- conf[h,c,:] = sum_{n: pseudo_n = c} preds[h,n,:], rows / max(sum, 1e-6)."""
    H, N, C = preds.shape
    sel = torch.nn.functional.one_hot(pseudo_labels, C).to(preds.dtype)        # (N, C)
    conf = torch.einsum("nc,hnj->hcj", sel, preds)
    return conf / conf.sum(-1, keepdim=True).clamp_min(1e-6)


def dirichlet_prior(conf: torch.Tensor, prior_strength: float, uniform: bool) -> torch.Tensor:
    """coda.py:46-63 -- base pseudo-counts + prior_strength * soft confusion."""
    H, C, _ = conf.shape
    if uniform:
        base = torch.full((C, C), 2 / C, dtype=conf.dtype)
    else:
        base = torch.full((C, C), 1.0 / (C - 1), dtype=conf.dtype)
        base.fill_diagonal_(1.0)
    return base.unsqueeze(0).expand(H, C, C) + prior_strength * conf


def consensus_marginals(dirichlets: torch.Tensor, preds: torch.Tensor):
    """coda.py:226-233 -- per-item and dataset-level consensus label marginals."""
    adj = torch.einsum("hcs,hns->hnc", dirichlets, preds)
    xi = adj.sum(0)
    xi = xi / xi.sum(dim=-1, keepdim=True).clamp_(min=1e-12)
    pi = xi.sum(0)
    pi = pi / pi.sum()
    return xi, pi


def pbest_rows(alpha: torch.Tensor, beta: torch.Tensor, nodes: int = QUAD_NODES,
               check: bool = True) -> torch.Tensor:
    """coda.py:77-119 -- P(model h has the largest Beta draw) for every row.

    alpha, beta: (R, H).  For each row: pdf on the grid (Beta.log_prob -> exp, 94-95),
    cumulative trapezoid cdf with cdf[0] = 0 (98-101), log(max(cdf, 1e-30)) (104),
    leave-one-out product exp(clamp(sum_h' L - L_h, -80, 80)) (107), trapz of
    pdf * product (108-111), normalise over h with a 1e-30 floor (114)."""
    R, H = alpha.shape
    x = quad_grid(nodes, alpha.device)
    # Beta.log_prob == Dirichlet([a, b]).log_prob([x, 1-x])
    #   (torch/distributions/beta.py:87-91, dirichlet.py:90-97)
    a = alpha.reshape(1, -1)
    b = beta.reshape(1, -1)
    xs = x.reshape(-1, 1)
    logpdf = (torch.xlogy(a - 1.0, xs) + torch.xlogy(b - 1.0, 1.0 - xs)) \
        + torch.lgamma(a + b) - (torch.lgamma(a) + torch.lgamma(b))           # (P, R*H)
    pdf = logpdf.exp().T.reshape(R, H, nodes)
    if check:
        _finite_or_raise(pdf, "pdf")
    cdf = torch.zeros_like(pdf)
    for j in range(1, nodes):                                                   # 99-101
        cdf[:, :, j] = cdf[:, :, j - 1] + 0.5 * (pdf[:, :, j] + pdf[:, :, j - 1]) * (x[j] - x[j - 1])
    if check:
        _finite_or_raise(cdf, "cdf")
    L = torch.log(cdf.clamp_min(CDF_FLOOR))
    loo = torch.exp((L.sum(1, keepdim=True) - L).clamp(-EXP_CLAMP, EXP_CLAMP))
    integrand = pdf * loo
    if check:
        _finite_or_raise(integrand, "integrand")
    prob = torch.trapz(integrand, x, dim=2)
    if check:
        _finite_or_raise(prob, "Pbest(beta)")
    prob = prob / prob.sum(-1, keepdim=True).clamp_min(CDF_FLOOR)
    if check:
        _finite_or_raise(prob, "Pbest(beta) normalized")
    return prob                                                                 # (R, H)


def hard_predictions(preds: torch.Tensor) -> torch.Tensor:
    """coda.py:263 / 316 -- argmax over classes, (H, N)."""
    return preds.argmax(-1)


def disagreement_mask(hard: torch.Tensor) -> torch.Tensor:
    """coda.py:215-219 -- keep points where at least one model differs from the majority vote
    (i.e. the models are not unanimous; trap T4)."""
    maj, _ = torch.mode(hard, dim=0)
    return (hard != maj).sum(0) > 0


def entropy2(p: torch.Tensor) -> torch.Tensor:
    """coda.py:254, 276 -- base-2 entropy with both factors clamped at 1e-12 (trap T7)."""
    q = p.clamp_min(ENT_FLOOR)
    return -(q * q.log2()).sum(-1)


class OracleSelector:
    """State + the three ``ModelSelector`` calls (coda/base.py:1-16), restated.

    Holds exactly the attributes callers read on the reference's ``CODA``
    (coda.py:181-203): dirichlets, pi_hat_xi, pi_hat, labeled_idxs, labels, q_vals,
    unlabeled_idxs, stochastic, step."""

    def __init__(self, preds: torch.Tensor, prefilter_n: int = 0, alpha: float = 0.9,
                 learning_rate: float = 0.01, multiplier: float = 2.0,
                 disable_diag_prior: bool = False, q: str = "eig", check: bool = True):
        assert preds.dtype == torch.float32 and preds.dim() == 3
        self.preds = preds
        self.H, self.N, self.C = preds.shape
        self.prefilter_n = prefilter_n
        self.q = q
        self.check = check
        self.prior_strength = 1 - alpha                                        # coda.py:189
        self.update_strength = learning_rate                                   # coda.py:190
        pseudo = preds.mean(dim=0).argmax(-1)                                  # coda.py:193-194, util.py:13-14
        conf = soft_confusion(pseudo, preds)                                   # coda.py:195
        self.dirichlets = multiplier * dirichlet_prior(conf, self.prior_strength, disable_diag_prior)  # 196
        self.hard = hard_predictions(preds)                                    # (H, N), reused below
        self.pi_hat_xi, self.pi_hat = consensus_marginals(self.dirichlets, preds)  # coda.py:197
        self.labeled_idxs, self.labels, self.q_vals = [], [], []
        self.unlabeled_idxs = list(range(self.N))
        self.stochastic = False
        self.step = 0

    # -- acquisition -----------------------------------------------------------------
    def candidates(self):
        """coda.py:215-224 + 239 -- non-unanimous unlabeled points, else all unlabeled."""
        mask = disagreement_mask(self.hard)
        keep = [i for i in self.unlabeled_idxs if mask[i]]
        if self.prefilter_n and len(keep) > self.prefilter_n:
            keep = _pyrandom.sample(keep, self.prefilter_n)
            self.stochastic = True
        return keep or self.unlabeled_idxs

    def pbest_before(self):
        """coda.py:245-251 -- P(best | class row c) under the current posterior, (C, H)."""
        a, b = diag_beta_params(self.dirichlets)                               # (H, C)
        return pbest_rows(a.T.contiguous(), b.T.contiguous(), check=self.check)

    def eig_scores(self, cand: list[int], chunk: int = CHUNK, w: float = HYP_WEIGHT) -> torch.Tensor:
        """coda.py:235-281 -- EIG of every candidate.

        For candidate b and hypothetical class c, every model's class-c Beta is
        updated as if the label were c: alpha += w where the model predicts c, beta += w
        where it does not (coda.py:150-168, trap T2: w is 1.0, not the learning rate);
        pi_hat is NOT hypothetically updated (trap T3)."""
        H, C = self.H, self.C
        a0, b0 = diag_beta_params(self.dirichlets)                             # (H, C)
        pb = self.pbest_before()                                               # (C, H)
        mix0 = (self.pi_hat[:, None] * pb).sum(0)                              # (H,)   coda.py:253
        h_before = entropy2(mix0)                                              # coda.py:254
        out = []
        cand_t = torch.tensor(cand, dtype=torch.long)
        for s in range(0, len(cand), chunk):
            ids = cand_t[s:s + chunk]
            B = ids.numel()
            hp = self.hard[:, ids].T                                           # (B, H)     coda.py:263
            hit = hp[:, :, None] == torch.arange(C)[None, None, :]             # (B, H, C)  coda.py:158-161
            a = a0[None].expand(B, H, C).clone()
            b = b0[None].expand(B, H, C).clone()
            a[hit] += 1.0 * w                                                  # coda.py:165
            b[~hit] += 1.0 * w                                                 # coda.py:166
            a = a.permute(0, 2, 1).reshape(B * C, H)                           # rows = (b, c)
            b = b.permute(0, 2, 1).reshape(B * C, H)
            ph = pbest_rows(a, b, check=self.check).reshape(B, C, H)           # coda.py:271
            mix = mix0[None, None, :] + self.pi_hat[None, :, None] * (ph - pb[None])   # coda.py:274-275
            h_after = entropy2(mix)                                            # (B, C)     coda.py:276
            out.append(h_before - (self.pi_hat_xi[ids] * h_after).sum(-1))     # coda.py:278
        return torch.cat(out) if out else torch.zeros(0)

    def get_next_item_to_label(self):
        """coda.py:283-313, including the two ablation acquisitions (coda.py:287-295)."""
        if self.q == "eig":
            cand = self.candidates()
            qv = self.eig_scores(cand)
        elif self.q == "iid":                                                   # coda.py:287-290
            cand = self.candidates()
            qv = 1 / len(cand) * torch.ones(len(cand))
        elif self.q == "uncertainty":                                           # coda.py:291-295, baselines/uncertainty.py:6-11
            cand = self.candidates()
            mean = self.preds.mean(dim=0)
            ent = -torch.sum(mean * torch.log(mean + 1e-8), dim=-1)
            qv = ent[cand]
        else:
            raise NotImplementedError(self.q)
        self.last_q, self.last_cand = qv, cand
        best = qv.max()
        ties = torch.isclose(qv, best, rtol=1e-8)                               # coda.py:307 (atol default 1e-8, trap T6)
        if int(ties.sum()) > 1:
            loc = _pyrandom.choice(torch.nonzero(ties, as_tuple=True)[0].tolist())
            self.stochastic = True
        else:
            loc = int(torch.argmax(qv))
        return cand[loc], float(qv[loc])

    # -- posterior update ------------------------------------------------------------
    def add_label(self, idx: int, true_class: int, selection_prob: float) -> None:
        """coda.py:315-323 -- D[h, true_class, p_h(idx)] += learning_rate, then refresh pi_hat."""
        onehot = torch.nn.functional.one_hot(self.hard[:, idx], self.C).float()
        self.dirichlets[:, true_class] += self.update_strength * onehot
        self.pi_hat_xi, self.pi_hat = consensus_marginals(self.dirichlets, self.preds)
        self.labeled_idxs.append(idx)
        self.labels.append(int(true_class))
        self.q_vals.append(selection_prob)
        self.unlabeled_idxs.remove(idx)

    def get_pbest(self) -> torch.Tensor:
        """coda.py:122-147, 325-332 -- pbest[h] = sum_c pi_hat[c] * P(best | row c)[h], shape (1, H)."""
        pb = self.pbest_before()
        out = (pb * self.pi_hat[:, None]).sum(0, keepdim=True)
        if self.check:
            _finite_or_raise(out, "Pbest")
        return out

    def get_best_model_prediction(self) -> torch.Tensor:
        """coda.py:334-346 -- increments ``step`` and returns a 0-d LongTensor (trap T10)."""
        pb = self.get_pbest()
        self.step += 1
        return torch.argmax(pb)


# ---------------------------------------------------------------------------------------
# bounded CPU-baseline samples for bench.py (SURVEY.md 8d, BASELINE.md section 3)
# ---------------------------------------------------------------------------------------
def time_step_sample(sel: OracleSelector, n_chunks: int, seed: int = 0):
    """Time the three pieces of one acquisition step on a bounded sample and extrapolate:
    ``n_chunks`` random 100-point chunks of the EIG loop (coda.py:262-279), one
    consensus_marginals refresh and one candidate prefilter, all on whatever slab ``sel``
    holds.  Returns seconds for (eig per chunk, marginals, prefilter)."""
    import time
    g = torch.Generator().manual_seed(seed)
    t0 = time.perf_counter()
    cand = sel.candidates()
    t_pref = time.perf_counter() - t0
    picks = torch.randperm(len(cand), generator=g)[: n_chunks * CHUNK].tolist()
    sub = sorted(cand[i] for i in picks)
    t0 = time.perf_counter()
    sel.eig_scores(sub)
    t_eig = (time.perf_counter() - t0) / max(1, (len(sub) + CHUNK - 1) // CHUNK)
    t0 = time.perf_counter()
    consensus_marginals(sel.dirichlets, sel.preds)
    t_pi = time.perf_counter() - t0
    return t_eig, t_pi, t_pref
