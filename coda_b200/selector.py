"""``CODA`` -- host-side mirror of the reference selector (coda/coda.py:171-346) over the sm_90a kernels.

Same constructor, same three ``ModelSelector`` calls, same attributes callers read
(``stochastic``, ``unlabeled_idxs``, ``pi_hat``, ``pi_hat_xi``, ``dirichlets``, ``labeled_idxs``,
``labels``, ``q_vals``, ``step``, ``H/N/C``, ``device``), same error types.  The arithmetic is in
``libcoda_b200.so``; there is no CPU route -- a CPU ``dataset.preds`` raises.

Sharding (SURVEY.md 8e), chosen at construction:
  * one process per GPU (torchrun + ``torch.distributed`` initialised): this process owns one shard;
  * ONE process, several GPUs (``main.py`` unchanged): ``gpus=`` / ``CODA_B200_GPUS`` (default: every visible GPU once the
    slab is >= 4 GiB) splits ``dataset.preds`` along N -- shard 0 reads the caller's tensor in place, the others get
    peer copies -- and this object drives all shards, each on its own stream;
  * ``shards=`` > number of GPUs puts several shards on one GPU (the 1-GPU test tier exercises the exchange that way).
"""
from __future__ import annotations

import math
import os
import random

import numpy as np
import torch

from .base import ModelSelector
from .dist import choose_among_ties, default_comm, labels_per_device, shard_layout
from .engine import HIST_CAP, TIE_CAP, build_engines


class _Unlabeled:
    """List-like view of the unlabeled item indices (coda.py:200, 323; demo/app.py:188 calls ``remove``).
    The reference keeps a Python list and pays O(N) per removal; this keeps a removed-set and a device mask."""

    def __init__(self, n_lo: int, n_hi: int, on_remove):
        self._lo, self._hi = n_lo, n_hi
        self._removed = set()
        self._on_remove = on_remove

    def remove(self, idx):
        idx = int(idx)
        if not (self._lo <= idx < self._hi) or idx in self._removed:
            raise ValueError("list.remove(x): x not in list")             # coda.py:323 behaviour
        self._removed.add(idx)
        self._on_remove(idx)

    def __contains__(self, idx):
        return self._lo <= int(idx) < self._hi and int(idx) not in self._removed

    def __len__(self):
        return self._hi - self._lo - len(self._removed)

    def __iter__(self):
        rem = self._removed
        return (i for i in range(self._lo, self._hi) if i not in rem)

    def __getitem__(self, k):
        return list(self)[k]


ABL_CHUNK_WORDS = 1 << 22      # int64 words of one shard's pre-draw buffer (q='iid' / prefilter_n device loop)


def candidate_counts(d0: int, u0: int, k: int):
    """The candidate count n_s of each of ``k`` steps from ``d0`` unlabeled items some model disagrees on and ``u0``
    unlabeled items: every pick removes one candidate, so n_s = d0 - s while that is > 0, then u0 - s (coda.py:239)."""
    return [d0 - s if d0 - s > 0 else u0 - s for s in range(k)]


def ablation_draw(kind: str, n: int, m: int = 0):
    """The Python ``random`` draws of one step with ``n`` candidates, made with the calls of the API path, as a pre-draw
    row: ``kind='iid'`` -> [n, k], k = ``random.choice`` over the n candidates (no draw for one candidate: the arg-max
    of coda.py:309); ``'prefilter'`` -> [n, positions...], ``random.sample`` of ``m`` positions into the ascending
    candidate list (called only when n > m).  ``random.choice(range(n))`` and ``random.sample(range(n), m)`` consume
    what the same calls on an n-item list consume and return its positions."""
    if kind == "iid":
        return [n, random.choice(range(n)) if n > 1 else 0]
    return [n] + random.sample(range(n), m)


def sample_setsize(m: int) -> int:
    """Lib/random.py's ``setsize`` of ``random.sample(population, m)``: a population of at most this many items is
    sampled from a list (pool branch), a larger one by rejecting repeats (set branch)."""
    setsize = 21
    if m > 5:
        setsize += 4 ** math.ceil(math.log(m * 3, 4))
    return setsize


def rng_words(state) -> torch.Tensor:
    """random.getstate() -> the device replica's int32 [625]: the 624 MT19937 words (as uint32 bits), the position."""
    return torch.from_numpy(np.array(state[1], dtype=np.uint32).view(np.int32).copy())


def rng_state(words: torch.Tensor, gauss_next):
    """The inverse of ``rng_words``: a state for random.setstate, with ``gauss_next`` as given."""
    return (3, tuple(int(w) for w in words.numpy().view(np.uint32)), gauss_next)


def _auto_gpus(preds) -> int:
    env = os.environ.get("CODA_B200_GPUS")
    if env:
        return max(1, int(env))
    nbytes = preds.numel() * (preds.element_size() if isinstance(preds, torch.Tensor) else 4)
    if nbytes < (4 << 30):
        return 1
    return max(1, torch.cuda.device_count())


class CODA(ModelSelector):
    def __init__(self, dataset, prefilter_n=0, alpha=0.9, learning_rate=0.01, multiplier=2.0,
                 disable_diag_prior=False, q="eig", *, mode="incremental", comm=None, gpus=None, shards=None):
        self.dataset = dataset
        preds = dataset.preds
        self.device = preds.device
        self.prefilter_n = prefilter_n
        self.disable_diag_prior = disable_diag_prior
        self.q = q
        self.prior_strength = 1 - alpha                     # coda.py:189
        self.update_strength = learning_rate                # coda.py:190
        comm = comm or default_comm()
        n_offset = int(getattr(dataset, "n_offset", 0))
        n_global = int(getattr(dataset, "n_global", preds.shape[1]))
        kw = dict(alpha=alpha, learning_rate=learning_rate, multiplier=multiplier,
                  uniform_prior=bool(disable_diag_prior), mode=mode, n_global=n_global, prefilter_n=prefilter_n, q=q)
        self.group, layout = shard_layout(preds, gpus, shards, comm, n_offset, default=lambda: _auto_gpus(preds))
        self.engines = build_engines(layout, self.group, **kw)
        self.engine = self.engines[0]
        self.H, self.C = self.engine.H, self.engine.C
        self.N = n_global                                   # callers see the whole task (coda.py:183)
        self.labeled_idxs, self.labels = [], []
        self.unlabeled_idxs = _Unlabeled(0, n_global, self._mark_labeled)
        self.q_vals = []
        self.stochastic = False
        self.step = 0
        self.last_report = None
        self._hist_seen = 0                                 # device-loop steps already mirrored into the host lists
        self._labels_dev = None
        self._loop_dirty = False

    @classmethod
    def from_args(cls, dataset, args):
        """coda.py:205-213"""
        return cls(dataset, prefilter_n=args.prefilter_n, alpha=args.alpha, learning_rate=args.learning_rate,
                   multiplier=args.multiplier, disable_diag_prior=args.no_diag_prior, q=args.q)

    # -- plumbing over the shards -----------------------------------------------------------------
    def _sync(self):
        for e in self.engines:
            e.sync()

    def _mark_labeled(self, idx):
        for e in self.engines:
            e.mark_labeled(idx)

    def _home(self, t):
        return t if t.device == self.device else t.to(self.device)

    def _cat(self, name):
        """Per-item vector ``name`` over all items, on the dataset's device (cold paths).  With one process per GPU it
        would need a host all-gather of N-sized vectors: not offered there -- use the single-process front end."""
        if self.group.world > 1 and len(self.engines) == 1:
            raise NotImplementedError("this acquisition variant needs all items in one process: build CODA with "
                                      "gpus=... (one process driving all GPUs) instead of one process per GPU")
        self._sync()
        if len(self.engines) == 1:
            return getattr(self.engine, name)
        return torch.cat([self._home(getattr(e, name)) for e in self.engines], 0)

    # -- attributes the reference exposes as tensors ---------------------------------------
    @property
    def dirichlets(self):
        self._sync()
        return self.engine.D

    @property
    def pi_hat(self):
        self._sync()
        return self.engine.pi_hat

    @property
    def pi_hat_xi(self):
        parts = [e.pi_hat_xi() for e in self.engines]
        self._sync()
        return parts[0] if len(parts) == 1 else torch.cat([self._home(p) for p in parts], 0)

    @property
    def eig(self):
        """Per-item expected information gain of the last scoring pass (this process's shards, item order).  When the
        engine scores only the ``prefilter_n`` sample (``sample_scoring``), an entry is current only for the items
        scored last; the others keep the value they were last scored with (0 if never)."""
        self._sync()
        return self.engine.eig if len(self.engines) == 1 else torch.cat([self._home(e.eig) for e in self.engines], 0)

    # -- acquisition -------------------------------------------------------------------------
    def _fetch_report(self):
        for e in self.engines:
            e.report()                                      # enqueue on every shard before anyone waits
        rep = self.engine.fetch()
        self.last_report = rep
        self.engine.check_flags(flags=rep["flags"])
        return rep

    def get_next_item_to_label(self):
        """coda.py:283-313.  Returns (global item index: int, q: float)."""
        if self.q in ("iid", "uncertainty"):
            return self._select_ablation()                  # coda.py:287-295
        if self.q != "eig":
            raise NotImplementedError(self.q)               # coda.py:297
        if self.prefilter_n:
            return self._select_prefiltered()
        rep = self._fetch_report()
        if rep["n_ties"] == 0:
            raise RuntimeError("no unlabeled items left to select from")
        if rep["n_ties"] > 1:                               # coda.py:308-311
            self.stochastic = True
            if rep["n_ties"] <= len(rep["tie_idx"]):
                ties = rep["tie_idx"]
                idx = choose_among_ties(ties, random)
                q = float(rep["tie_val"][int(np.nonzero(ties == idx)[0][0])])
            else:
                idx, q = self._select_many_ties(rep)
            return idx, q
        return int(rep["tie_idx"][0]), float(rep["tie_val"][0])   # == arg-max, first index wins (coda.py:309)

    @staticmethod
    def _candidate_mask(labeled, disagree):
        m = (labeled == 0) & (disagree != 0)
        if not bool(m.any()):
            m = labeled == 0                                # coda.py:239 `or self.unlabeled_idxs`
        return m

    def _select_ablation(self):
        """coda.py:287-295: the two ablation acquisitions of the paper (random / ensemble-entropy sampling) followed by
        the same tie rule (coda.py:306-313).  Cold path over ``ens`` = sum_h preds from the slab scan."""
        if self.prefilter_n:
            raise NotImplementedError(f"q={self.q!r} together with prefilter_n")
        mask = self._candidate_mask(self._cat("labeled"), self._cat("disagree"))
        n = int(mask.sum())
        if n == 0:
            raise RuntimeError("no unlabeled items left to select from")
        if self.q == "iid":
            qv = torch.full((self.N,), np.float32(1.0 / n).item(), dtype=torch.float32, device=self.device)
        else:
            if getattr(self, "_ens_entropy", None) is None:      # non-adaptive: computed once (uncertainty.py:6-11)
                if self.engine.ens is None:
                    raise RuntimeError("q='uncertainty' needs the ensemble sums (CODA_B200_ENS=0 disables them)")
                from .baselines import ensemble_entropy
                self._ens_entropy = ensemble_entropy(self._cat("ens"), self.H)
            qv = self._ens_entropy
        best = qv[mask].max()
        ties = torch.isclose(qv, best, rtol=1e-8) & mask        # coda.py:307
        nt = int(ties.sum())
        if nt > 1:                                              # coda.py:308-311
            idx = random.choice(torch.nonzero(ties, as_tuple=True)[0].tolist())
            self.stochastic = True
        else:
            idx = int(torch.nonzero(ties, as_tuple=True)[0][0])
        return idx, float(qv[idx])

    def _select_many_ties(self, rep):
        """More than TIE_CAP isclose-ties: evaluate the tie rule on the full vector (cold path)."""
        eig = self._cat("eig").cpu().numpy()
        cand = np.nonzero(self._candidate_mask(self._cat("labeled"), self._cat("disagree")).cpu().numpy())[0]
        qv = eig[cand]
        best = np.float32(rep["best_val"])
        tol = np.float32(1e-8) + np.abs(np.float32(1e-8) * best)
        ties = cand[(qv == best) | (np.abs(qv - best) <= tol)]
        idx = choose_among_ties(ties, random)
        return int(idx), float(eig[idx])

    def _select_prefiltered(self):
        """coda.py:221-223: random subsample of the candidates (``--prefilter-n``), then coda.py:306-313
        on the subsample in sample order.  With sample scoring only the candidates the reference scores (the sample,
        or the whole candidate list when it is not sampled) are scored; otherwise every item is."""
        sample = self.engine.sample_scoring
        if not sample:
            self._fetch_report()
        labeled, disagree = self._cat("labeled"), self._cat("disagree")
        m = (labeled == 0) & (disagree != 0)
        ids = torch.nonzero(m, as_tuple=True)[0].tolist()
        if self.prefilter_n and len(ids) > self.prefilter_n:
            ids = random.sample(ids, self.prefilter_n)
            self.stochastic = True
        if not ids:
            ids = torch.nonzero(labeled == 0, as_tuple=True)[0].tolist()
        if sample:
            ids_t = torch.tensor(ids, dtype=torch.int64)
            for e in self.engines:
                lo, hi = e.n_offset, e.n_offset + e.N
                e.score_items(ids_t[(ids_t >= lo) & (ids_t < hi)] - lo)
            for e in self.engines:
                e.sync()
                e.check_flags(sync=True)
        qv = self._cat("eig")[torch.tensor(ids, device=self.device)]
        best = qv.max()
        ties = torch.isclose(qv, best, rtol=1e-8)
        if int(ties.sum()) > 1:
            loc = random.choice(torch.nonzero(ties, as_tuple=True)[0].tolist())
            self.stochastic = True
        else:
            loc = int(torch.argmax(qv))
        return ids[loc], float(qv[loc])

    # -- posterior update --------------------------------------------------------------------
    def add_label(self, idx, true_class, selection_prob):
        """coda.py:315-323"""
        idx, true_class = int(idx), int(true_class)
        if self._loop_dirty:
            self.history()                                  # a device loop ran: bring the host-side lists up to date first
        if not (0 <= true_class < self.C):
            raise IndexError(f"index {true_class} is out of bounds for dimension 1 with size {self.C}")
        if idx not in self.unlabeled_idxs:
            raise ValueError("list.remove(x): x not in list")
        eager = self.q == "eig" and not self.prefilter_n    # the next call will want the scores: enqueue them now
        for e in self.engines:                              # phases in lock-step over the shards (see Engine.label_stage)
            e.label_stage(idx, true_class)
        if eager and all(e.api_graph_wanted() for e in self.engines):
            for e in self.engines:
                e.api_capture()
        for e in self.engines:
            e.label_run(eager)
        self.labeled_idxs.append(idx)
        self.labels.append(true_class)
        self.q_vals.append(selection_prob)
        self.unlabeled_idxs._removed.add(idx)               # the label kernels already set the device mask

    def get_pbest(self):
        """coda.py:325-332 -> (1, H) float32 tensor on the device."""
        out = self.engine.pbest()
        if self.engine.stream is not None:
            self.engine.sync()
        return out

    def get_best_model_prediction(self):
        """coda.py:334-346 -> a fresh 0-d LongTensor like torch.argmax (trap T10); bumps ``step``."""
        self.step += 1
        with self.engine._on():
            out = self.engine.best_model[0].clone()
        if self.engine.stream is not None:
            self.engine.sync()
        return out

    # -- host-free loop (SURVEY.md 8f rank 2) ----------------------------------------------------
    def _loop_refusals(self):
        """What the device loop does not offer, raised before anything is launched."""
        q = self.q
        if q not in ("eig", "iid", "uncertainty"):
            raise NotImplementedError(q)                    # coda.py:297
        if q == "eig" and not self.prefilter_n:
            return
        if q != "eig" and self.prefilter_n:
            raise NotImplementedError(f"q={q!r} together with prefilter_n")
        if self.group.world > 1 and len(self.engines) == 1:
            raise NotImplementedError("run_steps with q='iid' / 'uncertainty' or prefilter_n needs all items in one "
                                      "process: build CODA with gpus=... (one process driving all GPUs) instead of one "
                                      "process per GPU")
        if q == "uncertainty" and self.engine.ens is None:
            raise RuntimeError("q='uncertainty' needs the ensemble sums (CODA_B200_ENS=0 disables them)")

    def _reference_refusals(self):
        """What tie_rule="reference" does not offer, raised before anything is launched."""
        if self.group.world > 1 and len(self.engines) == 1:
            raise NotImplementedError("run_steps(tie_rule='reference') needs all items in one process: build CODA with "
                                      "gpus=... (one process driving all GPUs) instead of one process per GPU")
        inst = getattr(random, "_inst", None)
        if type(inst) is not random.Random:
            raise RuntimeError("tie_rule='reference' follows the random module's own generator, which has been "
                               f"replaced by a {type(inst).__name__}")
        if random.Random._randbelow is not random.Random._randbelow_with_getrandbits:
            raise RuntimeError("tie_rule='reference' needs random.Random._randbelow to be _randbelow_with_getrandbits")
        if self.N >= 2 ** 32:
            raise NotImplementedError("tie_rule='reference' draws _randbelow over candidate counts below 2**32")
        m = int(self.prefilter_n or 0)
        if m and len(self.engines) > 1:
            bound = int(self.engine.lib.coda_b200_pf_tie_max_m(self.H))
            if m > bound:
                raise NotImplementedError(f"tie_rule='reference' with {len(self.engines)} shards takes prefilter_n <= "
                                          f"{bound} at H={self.H} (the tie draw's sample bitmap travels in one record "
                                          f"slot); got {m}")

    def run_steps(self, k, labels, *, record_best=False, tie_rule="first"):
        """``k`` acquisition steps with the oracle's labels resident on the device(s): main.py:89-94 without a host
        round trip (arg-max pick, first index on equal values; a step where the reference would have drawn from
        ``random.choice`` because of an isclose tie is flagged in ``history()``).  ``labels``: int64 tensor of all N
        labels.  ``record_best``: replay a graph that also records every step's best model (``best_history()``, the
        regret curve of main.py:94-103); the default graph does not.  Returns nothing; read ``history()`` /
        ``get_pbest()`` afterwards.

        Runs the acquisition the selector was built with: ``q='uncertainty'`` and ``q='iid'`` (coda.py:287-295) and
        ``prefilter_n`` (coda.py:215-224) as well as EIG.  Their Python ``random`` draws (iid's ``random.choice``, the
        prefilter's ``random.sample``) do not depend on the data and are made on the host before the steps run, with
        the API path's own calls (DESIGN.md §4).

        ``tie_rule``: which random stream the picks follow.  ``"first"`` (the default) takes the first maximum of an
        isclose tie and only flags the step.  ``"reference"`` breaks it as coda.py:306-311 does, with ``random.choice``'s
        draw made on the device from a replica of Python's generator; the prefilter's samples come from the same
        replica.  Then the picks, q values, ``stochastic``, the posterior and the final ``random.getstate()`` are those
        of ``k`` API steps.  q='iid' draws before the loop either way."""
        if tie_rule not in ("first", "reference"):
            raise ValueError(f"tie_rule must be 'first' or 'reference', got {tie_rule!r}")
        self._loop_refusals()
        rule = "reference" if tie_rule == "reference" and self.q != "iid" else "first"
        if rule == "reference":
            self._reference_refusals()
        if self._labels_dev is None or self._labels_dev[0] is not labels:
            self._labels_dev = (labels, labels_per_device(labels, [e.dev for e in self.engines]))
        per_dev = self._labels_dev[1]
        if k <= 0:
            return
        if rule == "reference":
            self._run_reference(k, per_dev, record_best)
        elif self.q != "eig" or self.prefilter_n:
            self._run_ablation(k, per_dev, record_best)
        else:
            self._steps("eig", k, per_dev, record_best)

    def _run_reference(self, k, per_dev, record_best):
        """run_steps(tie_rule="reference"): Python's state goes to every shard's replica before the steps and comes
        back from it after them."""
        e0 = self.engine
        with e0._on():
            ctr0 = int(e0.step_ctr.item())
        words = rng_words(random.getstate())
        for e in self.engines:
            e.ref_bind()
            e.rng_upload(words)
        if self.q == "eig" and not self.prefilter_n:
            self._steps("eig", k, per_dev, record_best, "reference")
        else:
            self._run_ablation(k, per_dev, record_best, "reference")
        states = [e.rng_download() for e in self.engines]
        if any(not torch.equal(s, states[0]) for s in states[1:]):
            raise RuntimeError("the shards' replicas of Python's generator differ after run_steps")
        random.setstate(rng_state(states[0], random.getstate()[2]))
        with e0._on():
            slots = torch.arange(ctr0, int(e0.step_ctr.item()), device=e0.dev) % HIST_CAP
            if bool(e0.hist_tie[slots].any()):
                self.stochastic = True                      # coda.py:311

    def _steps(self, kind, k, per_dev, record_best, rule="first"):
        """``k`` steps of the loop body ``kind`` (engine.py, "host-free loop") on every shard.  Phases in lock-step over
        the shards, so that nobody waits on the host for a peer that has not been enqueued: prepare, then -- when a
        graph is missing -- one eager step (module loading outside the capture) and the capture, then replays."""
        self._loop_dirty = True
        for e in self.engines:
            e.loop_prepare(per_dev[e.dev], record_best, kind)
        if not all(e.loop_ready(record_best, rule, kind) for e in self.engines):
            for e in self.engines:
                e.loop_eager(record_best, rule, kind)
            k -= 1
            for e in self.engines:
                e.loop_capture(record_best, rule, kind)
        for _ in range(k):
            for e in self.engines:
                e.loop_replay(1, record_best, rule, kind)

    def _run_ablation(self, k, per_dev, record_best, rule="first"):
        """run_steps for q='uncertainty' / 'iid' / prefilter_n (the loop kinds of engine.py's host-free loop)."""
        d0 = u0 = 0
        for e in self.engines:                              # the candidate counts once; every step removes a candidate
            d, u = e.candidate_counts()
            d0, u0 = d0 + d, u0 + u
        if k > u0:
            raise RuntimeError("no unlabeled items left to select from")
        kind = "prefilter" if self.q == "eig" else self.q
        if kind == "uncertainty":
            if getattr(self, "_ens_entropy", None) is None:  # the API path's vector (see _select_ablation)
                from .baselines import ensemble_entropy
                self._ens_entropy = ensemble_entropy(self._cat("ens"), self.H)
            base = self.engines[0].n_offset
            for e in self.engines:
                e.abl_bind(kind, score=self._ens_entropy[e.n_offset - base: e.n_offset - base + e.N])
            self._steps(kind, k, per_dev, record_best, rule)
            return
        m = int(self.prefilter_n)
        counts = candidate_counts(d0, u0, k)
        # iid: every step; prefilter: the steps with more disagreeing candidates than the sample (a prefix: their count
        # falls by one per step), the rest -- the all-unlabeled fallback included -- are the plain arg-max of the EIG loop
        drawn = k if kind == "iid" else max(0, min(k, d0 - m))
        width = 2 if kind == "iid" else m + 1
        rows = max(1, ABL_CHUNK_WORDS // width)
        if drawn and rule == "reference":                   # the device samples each step's row itself
            for e in self.engines:
                e.abl_bind(kind, width=width, rows=1)
                e.ref_bind_prefilter(m, sample_setsize(m))
            self._steps(kind, drawn, per_dev, record_best, rule)
            self.stochastic = True                          # coda.py:223
        elif drawn:
            for e in self.engines:
                e.abl_bind(kind, width=width, rows=rows)
            for s0 in range(0, drawn, rows):
                c = min(rows, drawn - s0)
                pre = torch.tensor([ablation_draw(kind, counts[s0 + i], m) for i in range(c)], dtype=torch.int64)
                pre = pre.reshape(-1).pin_memory()
                for e in self.engines:
                    e.abl_load(pre)
                self._steps(kind, c, per_dev, record_best)
            if kind == "prefilter" or any(n > 1 for n in counts):
                self.stochastic = True                      # coda.py:223 / 311
        if k > drawn and kind == "prefilter" and self.engine.sample_scoring:
            self._run_unsampled(counts, drawn, k, m, per_dev, record_best, rule)
        elif k > drawn:
            self._steps("eig", k - drawn, per_dev, record_best, rule)

    def _run_unsampled(self, counts, s, k, m, per_dev, record_best, rule):
        """Sample scoring, the prefilter steps without a sample (n_s <= prefilter_n, or the all-unlabeled fallback):
        every candidate is scored.  Up to m candidates run the prefilter's graph with the identity sample
        (k_pf_identity: all candidates in ascending order, no random draw, so the pick, q and tie flag of the EIG
        loop); more, which only the fallback has, run eagerly with every item scored in chunks of m."""
        width = m + 1
        for e in self.engines:
            e.abl_bind("prefilter", width=width, rows=max(1, ABL_CHUNK_WORDS // width) if rule == "first" else 1)
            if rule == "reference":
                e.ref_bind_prefilter(m, sample_setsize(m))
        self._loop_dirty = True
        while s < k:
            big = counts[s] > m
            t = s
            while t < k and (counts[t] > m) == big:
                t += 1
            if big:
                for e in self.engines:
                    e.loop_prepare(per_dev[e.dev], record_best, "prefilter_id")   # labels and hist_best
                for _ in range(t - s):
                    for e in self.engines:
                        e.pf_fallback_score()
                    for e in self.engines:
                        e.pf_fallback_commit(rule, record_best)
            else:
                self._steps("prefilter_id", t - s, per_dev, record_best, rule)
            s = t

    def history(self):
        """(idx, q, tie) arrays of the device-loop steps so far (the last HIST_CAP of them); also mirrors them into the
        host-side bookkeeping the API path keeps (``labeled_idxs``, ``labels``, ``q_vals``, ``unlabeled_idxs``)."""
        self._sync()
        e = self.engine
        with e._on():
            n = int(e.step_ctr.item())
            idx = e.hist_idx[:n].cpu().numpy()
            q = e.hist_q[:n].cpu().numpy()
            tie = e.hist_tie[:n].cpu().numpy()
            e.check_flags(sync=True)
        if n > self._hist_seen and self._labels_dev is not None:
            lab = self._labels_dev[0]
            new = idx[self._hist_seen:n]
            cls = lab[torch.as_tensor(new, device=lab.device)].cpu().tolist() if len(new) else []
            for i, qq, t in zip(new.tolist(), q[self._hist_seen:n].tolist(), cls):
                self.labeled_idxs.append(int(i)); self.labels.append(int(t)); self.q_vals.append(float(qq))
                self.unlabeled_idxs._removed.add(int(i))
            self._hist_seen = n
        self._loop_dirty = False
        return idx, q, tie

    def best_history(self):
        """(best, best_tie) of the device-loop steps so far: the model ``get_best_model_prediction()`` returns after
        each step (-1 for a step run without ``record_best``), and ``best_tie``, always 0 (the best model is
        torch.argmax's first index, coda.py:346, in the reference too).  Also does what ``history()`` does."""
        idx, _q, _tie = self.history()
        n = len(idx)
        e = self.engine
        hb = getattr(e, "hist_best", None)
        with e._on():
            best = hb[:n].cpu().numpy() if hb is not None else np.full(n, -1, np.int32)
        return best, np.zeros(n, np.int32)

    # -- checkpoint / resume (SURVEY.md 8f rank 4; the reference restarts a killed seed from step 0) ------
    def state_dict(self):
        self._sync()
        sd = {"version": 1, "H": self.H, "N": self.N, "C": self.C, "mode": self.engine.mode,
              "labeled_idxs": list(self.labeled_idxs), "labels": list(self.labels), "q_vals": list(self.q_vals),
              "removed": sorted(self.unlabeled_idxs._removed), "stochastic": self.stochastic, "step": self.step,
              "python_random_state": random.getstate(), "shards": []}
        for e in self.engines:
            with e._on():
                sd["shards"].append({"n_offset": e.n_offset, "N": e.N,
                                     **{k: v.detach().cpu().clone() for k, v in e.state_tensors().items()}})
        return sd

    def load_state_dict(self, sd, restore_rng=True):
        """Resume a selector built on the same slab: bit-exact continuation (same picks, same posterior bits).
        The state may have been saved with a different shard count (this process must hold all its items)."""
        if (sd["H"], sd["N"], sd["C"]) != (self.H, self.N, self.C):
            raise ValueError("state_dict belongs to a different task shape")
        self._sync()
        order = sorted(sd["shards"], key=lambda s: s["n_offset"])
        U = torch.cat([s["U"] for s in order], 0)
        labeled = torch.cat([s["labeled"] for s in order], 0)
        base = order[0]["n_offset"]
        for e in self.engines:
            with e._on():
                lo, hi = e.n_offset - base, e.n_offset - base + e.N
                if lo < 0 or hi > U.shape[0]:
                    raise ValueError("state_dict does not cover this shard's items")
                e.D.copy_(order[0]["D"].to(e.dev))
                e.U.copy_(U[lo:hi].to(e.dev))
                e.labeled.copy_(labeled[lo:hi].to(e.dev))
                e.step_ctr.copy_(order[0]["step_ctr"].to(e.dev))
                e.pisum.zero_()
                e._call("coda_b200_pi_reduce", e.U.data_ptr(), e.N, e.C, e.fx_shift, None, e.pisum.data_ptr(),
                        e.flags.data_ptr(), e._s())
                e._tables(0, e.C)
                e.cache_valid, e.scored, e.reported, e.pending = False, False, False, False
                e.graphs.clear()
        for e in self.engines:
            e.construct_mixture()
        self._sync()
        self.labeled_idxs, self.labels, self.q_vals = list(sd["labeled_idxs"]), list(sd["labels"]), list(sd["q_vals"])
        self.unlabeled_idxs._removed = set(sd["removed"])
        self.stochastic, self.step = bool(sd["stochastic"]), int(sd["step"])
        if restore_rng:
            random.setstate(sd["python_random_state"])

    def close(self):
        """Free the device memory of every shard now (a selector is otherwise kept alive by reference cycles until gc)."""
        for e in self.engines:
            e.close()
        self._labels_dev = None
        self.dataset = None
