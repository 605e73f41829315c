"""tests/simref_leave.py's graceful leave and rejoin rules (ClusterSimulation.leave / rejoin) held to ClusterTest's own assertions
(testLeaving, testRejoinSingleNode, testRejoinSingleNodeSameConfiguration, testRejoinMultipleNodes, ClusterTest.java:417-521),
with the real ping-pong detectors raising the alerts.  The scenarios live in leave_scenarios.py;
test_gpu_cluster_leave_rejoin.py runs them on the device driver too and compares the runs."""
import pytest

import leave_scenarios as S

INTERVAL_KEYS = ("cfg", "interval", "alerts", "cells", "announced", "event", "leavers")


def records(s):
    return [{k: r[k] for k in INTERVAL_KEYS} for r in s.intervals], s.history


def test_leaving(orc):
    (s,) = S.leaving(orc, None)
    r = s.intervals[-1]
    assert r["leavers"] == 1 and r["event"] == "decided-fast" and r["announced"] == 10     # the remaining 10 agree
    assert r["alerts"] == 10                                                               # K LeaveMessages of live observers


def test_rejoin_single_node(orc):
    (s,) = S.rejoin_single_node(orc, None)
    assert [h["cut"] for h in s.history] == [[3]] * 4 and [h["size"] for h in s.history] == [9, 10, 9, 10]
    assert len({h["cfg_after"] for h in s.history} | {s.history[0]["cfg_before"]}) == 5    # a new NodeId: a new configuration


def test_rejoin_single_node_same_configuration(orc):
    (a,) = S.rejoin_same_configuration(orc, None)
    (b,) = S.rejoin_same_configuration(orc, None, refuse=False)
    assert records(a) == records(b)                                                        # the refusal changed nothing


@pytest.mark.parametrize("mode", ["crash", "leave"])
def test_rejoin_multiple_nodes(orc, mode):
    (s,) = S.rejoin_multiple_nodes(orc, None, mode)
    assert len(s.history) >= 6
    if mode == "leave":                                # every round's leave is decided in the interval the five leave in
        first = [r for r in s.intervals if r["leavers"]]
        assert len(first) == 3 and all(r["leavers"] == 5 and r["interval"] == 0 for r in first)


@pytest.mark.parametrize("how", ["leave", "crash"])
def test_leave_against_crash_on_the_same_draw(orc, how):
    S.leave_against_crash(orc, None, how)


def test_adjacent_leavers(orc):
    (s,) = S.adjacent_leavers(orc, None)
    assert s.intervals[0]["leavers"] == 2


def test_leaver_whose_observers_crashed(orc):
    S.leaver_with_crashed_observers(orc, None)


def test_refusals_change_nothing(orc):
    (a,) = S.refusals(orc, None)
    (b,) = S.refusals(orc, None, refuse=False)
    assert records(a) == records(b)


@pytest.mark.parametrize("seed", [13, 39])
def test_without_leaves_the_subclass_is_simref(orc, seed):
    """LeaveRejoinSimulation without leaves or rejoins runs exactly as simref's OracleSimulation (crashes while ten nodes join),
    with leavers 0 in every record"""
    from simref import OracleSimulation
    from simref_leave import LeaveRejoinSimulation
    n, nj = 30, 10
    a, b = (cls(orc, n, seed=seed, n_joiners=nj) for cls in (OracleSimulation, LeaveRejoinSimulation))
    for s in (a, b):
        S.flags((s,), range(2, 7), S.CRASHED)
        s.addJoiners(range(n, n + nj))
        assert s.run(30)["converged"]
    keys = INTERVAL_KEYS[:-1]
    assert [{k: r[k] for k in keys} for r in b.intervals] == [{k: r[k] for k in keys} for r in a.intervals]
    assert b.history == a.history and b.members == a.members
    assert all(r["leavers"] == 0 for r in b.intervals)
