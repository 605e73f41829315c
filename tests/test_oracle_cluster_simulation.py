"""tests/simref.py — ClusterSimulation's rules over the oracle's pieces — pinned against ClusterTest's own assertions
(ClusterTest.java:212-362, waitAndVerifyAgreement :710-730) on the scenarios of test_oracle_cluster_scenarios.py, this time
with the real ping-pong detectors (FdSim) raising the alerts, joins through the failure-detector interval, the seeded
fallback and the configuration-by-configuration view change.  test_gpu_cluster_simulation.py checks the device driver
against the same runs."""
import pytest

from simref import CRASHED, OracleSimulation, flags, random_hosts

INGRESS_BLOCKED = 2


def test_one_failure_out_of_five_nodes(orc):                                     # ClusterTest.java:212-224
    s = OracleSimulation(orc, 5, seed=1)
    flags((s,), [2], CRASHED)
    out = s.run(20)
    assert out["converged"] and s.members() == [0, 1, 3, 4]
    assert [h["path"] for h in s.history] == ["fast"] and s.history[0]["cut"] == [2]
    assert s.history[0]["intervals"] == 11                                        # ten failed probes, the notification on the 11th


@pytest.mark.parametrize("seed", [3, 4, 5])
def test_fail_random_quarter_of_nodes(orc, seed):                                # :275-291
    n, f = 50, 12
    failing = random_hosts(n, f, seed)
    s = OracleSimulation(orc, n, seed=seed)
    flags((s,), failing, CRASHED)
    out = s.run(30)
    assert out["converged"] and s.members() == [m for m in range(n) if m not in failing]
    assert s.view.getMembershipSize() == n - f
    assert sorted(t for h in s.history for t in h["cut"]) == failing


@pytest.mark.parametrize("seed", [6, 7, 8])
def test_fail_random_third_of_nodes(orc, seed):                                  # :299-315
    n, f = 50, 16
    failing = random_hosts(n, f, seed)
    s = OracleSimulation(orc, n, seed=seed)
    flags((s,), failing, CRASHED)
    out = s.run(30)
    assert out["converged"] and s.members() == [m for m in range(n) if m not in failing]
    assert s.history[0]["path"] == "classic"                                     # 34 voters < 38: the fallback decides
    assert all(h["distinct_proposals"] >= 1 for h in s.history)


@pytest.mark.parametrize("seed", [9, 10])
def test_fail_ten_random_nodes_that_stay_alive(orc, seed):                       # :322-336
    n, f = 50, 10
    failing = random_hosts(n, f, seed)
    s = OracleSimulation(orc, n, seed=seed)
    flags((s,), failing, INGRESS_BLOCKED)                                        # alive and voting; nobody answers their probes
    out = s.run(30)
    assert out["converged"] and s.members() == [m for m in range(n) if m not in failing]
    assert all(h["path"] == "fast" for h in s.history)


@pytest.mark.parametrize("seed", [13, 14, 15])
def test_concurrent_node_joins_and_fails(orc, seed):                             # :228-243
    n, f, nj = 30, 5, 10
    failing = list(range(2, 2 + f))
    joiners = list(range(n, n + nj))
    s = OracleSimulation(orc, n, seed=seed, n_joiners=nj)
    flags((s,), failing, CRASHED)
    s.addJoiners(joiners)
    out = s.run(30)
    assert out["converged"]
    assert sorted(s.members()) == sorted([m for m in range(n) if m not in failing] + joiners)
    assert s.view.getMembershipSize() == n - f + nj
    assert all(h["distinct_proposals"] >= 1 for h in s.history)


def test_inject_asymmetric_drops(orc):                                           # :342-360
    n, f = 50, 10
    failing = random_hosts(n, f, seed=12, lo=1)
    s = OracleSimulation(orc, n, seed=12)
    flags((s,), failing, INGRESS_BLOCKED)
    for _ in range(10):
        assert s.interval()["event"] == "quiet"
    flags((s,), failing, 0)                                                      # the drops end; the detectors have counted ten
    while not s.history:
        assert s.interval()["event"] != "stalled" and s.i < 5
    assert s.history[0]["cut"] == failing and s.history[0]["path"] == "fast"
    assert s.members() == [m for m in range(n) if m not in failing]


def test_edge_failures_cut_a_live_node(orc):
    """every observer of a live node fails its probes to it (per-edge failures, not node flags): ten failed probes, the alerts
    on the eleventh interval, and the node is cut on the fast path while every process is alive"""
    n, y = 50, 7
    s = OracleSimulation(orc, n, seed=16)
    for k, o in enumerate(s.view.getObserversOf(y)):
        s.setEdgeFail(o, k)
    while not s.history:
        assert s.interval()["event"] != "stalled" and s.i < 15
    assert s.history[0]["cut"] == [y] and s.history[0]["path"] == "fast" and s.history[0]["intervals"] == 11
    assert s.members() == [m for m in range(n) if m != y]


def test_a_third_of_the_nodes_can_block_the_cut(orc):
    """the draw of test_oracle_cluster_scenarios.py in which no live node ever proposes: the run reports the stall and the
    subjects it waits on instead of looping"""
    n, f, seed = 50, 16, 131
    failing = random_hosts(n, f, seed)
    s = OracleSimulation(orc, n, seed=seed)
    flags((s,), failing, CRASHED)
    out = s.run(15)
    assert out["stalled"] and not out["converged"] and out["stuck"] == failing
    assert s.history == [] and out["intervals"] == 15
    assert all(r["announced"] == 0 for r in s.intervals)
