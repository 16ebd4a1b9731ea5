"""CPU checks of CODA's device loop for q='iid' / q='uncertainty' / prefilter_n: the host pre-draws against the API
path's own calls, the candidate-count prediction against a simulation of the API loop, and the new ABI entries."""
import os
import random
import re

import numpy as np
import pytest

from helpers import ROOT


@pytest.mark.parametrize("n,m", [(10, 3), (25, 24), (5000, 7), (70, 60), (400, 5)])   # sample's pool and set branches
def test_prefilter_draw_matches_random_sample_over_the_candidate_list(n, m):
    from coda_b200.selector import ablation_draw
    ids = sorted(random.Random(n).sample(range(10 * n), n))        # any ascending candidate list
    random.seed(n * 31 + m)
    want = random.sample(ids, m)
    st = random.getstate()
    random.seed(n * 31 + m)
    row = ablation_draw("prefilter", n, m)
    assert random.getstate() == st
    assert row[0] == n and [ids[p] for p in row[1:]] == want


@pytest.mark.parametrize("n", [1, 2, 3, 17, 1000, 2 ** 20 + 5])
def test_iid_draw_matches_random_choice_over_the_candidate_list(n):
    from coda_b200.selector import ablation_draw
    ids = range(7, 7 + 3 * n, 3)
    random.seed(n)
    want = random.choice(list(ids)) if n > 1 else ids[0]           # one candidate: the arg-max, no draw
    st = random.getstate()
    random.seed(n)
    row = ablation_draw("iid", n)
    assert random.getstate() == st and row[0] == n and ids[row[1]] == want


@pytest.mark.parametrize("seed", range(4))
def test_candidate_count_prediction_follows_a_simulated_api_loop(seed):
    """The API loop on labeled / disagree masks: candidates are the unlabeled disagreeing items, all unlabeled items
    when there are none (coda.py:239); any candidate is picked.  Its counts equal candidate_counts(D0, U0, k)."""
    from coda_b200.selector import candidate_counts
    rng = np.random.default_rng(seed)
    N = 60
    disagree = rng.random(N) < 0.3
    labeled = rng.random(N) < 0.2
    d0, u0 = int((~labeled & disagree).sum()), int((~labeled).sum())
    seen = []
    for _ in range(u0):
        m = ~labeled & disagree
        if not m.any():
            m = ~labeled
        seen.append(int(m.sum()))
        labeled[rng.choice(np.nonzero(m)[0])] = True
    assert seen == candidate_counts(d0, u0, u0)


def test_new_abi_entries_and_their_argument_counts():
    from coda_b200 import _native as nat
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "coda_b200.h")).read(), flags=re.S)
    want = {"coda_b200_static_records": 8, "coda_b200_abl_draw": 4, "coda_b200_abl_commit": 7,
            "coda_b200_prefilter_blocks": 1, "coda_b200_prefilter_pick": 13, "coda_b200_prefilter_commit": 9}
    for name, n in want.items():
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", hdr, flags=re.S)
        assert m and m.group(1).count(",") + 1 == n == len(nat.SIGNATURES[name][1]), name
    assert nat.FLAG_PREDRAW_MISMATCH == 0x800 and "CODA_B200_FLAG_PREDRAW_MISMATCH 0x800u" in hdr
    assert nat.load().coda_b200_prefilter_blocks(17) == 3
