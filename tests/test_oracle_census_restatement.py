"""tests/censusref.py — ClusterSimulation's proposal census restated over simref's per-tag proposals — on oracle runs alone: the
records add up (voters to announcers, classes to distinct proposals, each configuration's classes to its intervals'), the decided
proposal is the cut, and the scenarios show what the census is for (three cuts in the shuffled 12-crash draw, joiners as UP
entries)."""
import pytest

import censusref
from simref import CRASHED, flags, join, leave, random_hosts, run


def sim(orc, n, seed, nj=0, **kw):
    return censusref.CensusOracleSimulation(orc, n, seed=seed, n_joiners=nj, **kw)


def consistent(s):
    for r in s.intervals:
        assert ("census" in r) == (r["announced"] > 0)
        if "census" in r:
            assert sum(c["voters"] for c in r["census"]) == r["announced"] and len(r["census"]) == r["proposals"]
            assert all(c["down"] + c["up"] == c["size"] for c in r["census"])
            assert len({c["representative"] for c in r["census"]}) == len(r["census"])
    for h in s.history:
        cls = h["census"]
        assert sum(c["voters"] for c in cls) == h["announced"] and len(cls) == h["distinct_proposals"]
        cfg_intervals = [r for r in s.intervals if r["cfg"] == h["cfg_before"] and "census" in r]
        assert sum(c["voters"] for r in cfg_intervals for c in r["census"]) == h["announced"]
        decided = [c for c in cls if c["decided"]]
        assert len(decided) == 1 and decided[0]["missing"] == decided[0]["extra"] == 0 and decided[0]["size"] == len(h["cut"])
        assert h["agreement"] == decided[0]["voters"] / h["announced"]
        for c in cls:
            assert c["size"] - c["extra"] == len(h["cut"]) - c["missing"]          # both count the proposal's nodes in the cut
    return s


@pytest.mark.parametrize("batch_order", ["sender", "shuffled"])
@pytest.mark.parametrize("n,f,seed", [(5, 1, 1), (50, 12, 3), (50, 16, 6)])
def test_failure_scenarios(orc, batch_order, n, f, seed):
    s = sim(orc, n, seed, batch_order=batch_order)
    flags((s,), [2] if n == 5 else random_hosts(n, f, seed), CRASHED)
    run((s,), 30)
    consistent(s)


def test_three_cuts_in_the_shuffled_draw(orc):
    s = sim(orc, 50, 12, batch_order="shuffled")
    flags((s,), random_hosts(50, 12, 12), CRASHED)
    run((s,), 30)
    consistent(s)
    h = s.history[0]
    assert len(h["census"]) == 3 and h["path"] == "classic" and 0 < h["agreement"] < 1
    assert sum(c["decided"] for c in h["census"]) == 1


def test_joiners_are_up_entries(orc):
    n, nj = 30, 10
    s = sim(orc, n, 13, nj)
    join((s,), range(n, n + nj))
    flags((s,), range(2, 7), CRASHED)
    run((s,), 30)
    consistent(s)
    ups = [c["up"] for h in s.history for c in h["census"] if c["decided"]]
    assert sum(ups) == nj


def test_graceful_leave(orc):
    s = sim(orc, 50, 31, batch_order="shuffled")
    leave((s,), [4, 17])
    run((s,), 30)
    consistent(s)
    assert sum(c["down"] for c in s.history[0]["census"] if c["decided"]) >= 2
