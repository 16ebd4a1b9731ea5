"""CPU checks of the sampled prefilter scoring: the new C entry points and their arity, and the scoring choice."""
import re

import pytest

from helpers import ROOT


NEW = {"coda_b200_pf_resolve": 11, "coda_b200_pf_identity": 6, "coda_b200_sample_plan": 15, "coda_b200_sample_fill": 15,
       "coda_b200_sample_gains": 12, "coda_b200_sample_eig": 15}


def test_new_entry_points_are_declared_bound_and_exported():
    from coda_b200 import _native as nat
    header = open(f"{ROOT}/include/coda_b200.h").read()
    lib = nat.load()
    for name, n in NEW.items():
        m = re.search(rf"int {name}\(([^;]*)\);", header)
        assert m, name
        assert len(m.group(1).split(",")) == n
        assert len(getattr(lib, name).argtypes) == n
    assert nat.VERSION == 203
    assert len(nat.load().coda_b200_prefilter_pick.argtypes) == 13


def test_scoring_choice_constants():
    from coda_b200 import engine
    assert engine.PREFILTER_SCORING == ("auto", "sample", "full")
    assert engine.PREFILTER_ROW_COST_RATIO > 0


@pytest.mark.parametrize("side", [0, 1])
def test_auto_rule(side):
    """auto: the sample when prefilter_n * R <= N (incremental mode, q='eig'); m just below / above N / R."""
    from coda_b200 import engine
    n = 100_000
    m = int(n / engine.PREFILTER_ROW_COST_RATIO) + side
    want = side == 0

    class E:
        pf_m, pf_scoring, mode, n_global = m, "auto", "incremental", n
    assert engine.Engine._choose_sample_scoring(E()) == (m * engine.PREFILTER_ROW_COST_RATIO <= n) == want
    E.mode = "recompute"
    assert not engine.Engine._choose_sample_scoring(E())
    E.mode, E.pf_scoring = "incremental", "full"
    assert not engine.Engine._choose_sample_scoring(E())
    E.pf_scoring = "sample"
    assert engine.Engine._choose_sample_scoring(E())
