"""tests/simref.py's graceful leave and rejoin rules (ClusterSimulation.leave / rejoin) held to ClusterTest's own assertions
(testLeaving, testRejoinSingleNode, testRejoinSingleNodeSameConfiguration, testRejoinMultipleNodes, ClusterTest.java:417-521),
with the real ping-pong detectors raising the alerts.  The scenarios live in leave_scenarios.py;
test_gpu_cluster_leave_rejoin.py runs them on the device driver too and compares the runs."""
import pytest

import leave_scenarios as S


def records(s):
    return s.intervals, s.history


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

