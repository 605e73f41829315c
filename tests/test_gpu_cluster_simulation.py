"""ClusterSimulation (rapid_b200/simulation.py) on the device against tests/simref.py — the same rules over the oracle's
pieces — configuration by configuration and interval by interval on ClusterTest's scenarios; the three device primitives it
adds (join alerts in the failure-detector interval, locating a proposer of a value, silent acceptors) on their own; and whole
failure scenarios at 10^4 (against simref), 10^5 and 10^6 nodes (against analytic expectations).

Above 10^4 nodes the runs are checked on their outcome only (membership, cuts, paths, the interval of each decision), not
receiver by receiver against an oracle window: the deciding interval's cut-detector state is replaced by the view change inside
interval(), and replaying 10^4-10^5 sender batches through the oracle per interval is beyond a test's time.  Receiver-level
parity of the same kernels at these sizes is held by test_gpu_cut_detection.py, test_gpu_full_scale.py and test_gpu_tally_cd.py,
and of the whole driver by the 10^4-node comparison with simref here."""
import numpy as np
import pytest

from simref import CRASHED, flags, join, make, random_hosts, run, same_run
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu

INGRESS_BLOCKED = 2


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


# ---- ClusterTest's scenarios, device vs simref ---------------------------------------------------------------------------------
def test_one_failure_out_of_five_nodes(orc, rb):
    ref, dev = sims = make(orc, rb, 5, 1)
    flags(sims, [2], CRASHED)
    run(sims, 20)
    same_run(ref, dev)
    assert dev.members() == [0, 1, 3, 4] and [h["path"] for h in dev.history] == ["fast"]


@pytest.mark.parametrize("n,f,seed,flag", [(50, 12, 3, CRASHED), (50, 12, 4, CRASHED), (50, 12, 5, CRASHED),
                                            (50, 16, 6, CRASHED), (50, 16, 7, CRASHED), (50, 16, 8, CRASHED),
                                            (50, 10, 9, INGRESS_BLOCKED), (50, 10, 10, INGRESS_BLOCKED)])
def test_failure_scenarios(orc, rb, n, f, seed, flag):                            # ClusterTest.java:275-336
    failing = random_hosts(n, f, seed)
    ref, dev = sims = make(orc, rb, n, seed)
    flags(sims, failing, flag)
    run(sims)
    same_run(ref, dev)
    assert dev.members() == [m for m in range(n) if m not in failing]
    if f == 16:
        assert dev.history[0]["path"] == "classic"                               # 34 voters < 38


@pytest.mark.parametrize("seed", [13, 14, 15])
def test_concurrent_node_joins_and_fails(orc, rb, seed):                         # :228-243
    n, nj = 30, 10
    ref, dev = sims = make(orc, rb, n, seed, n_joiners=nj)
    join(sims, range(n, n + nj))
    flags(sims, range(2, 7), CRASHED)
    run(sims)
    same_run(ref, dev)
    assert sorted(dev.members()) == sorted([m for m in range(n) if not 2 <= m < 7] + list(range(n, n + nj)))


def test_inject_asymmetric_drops(orc, rb):                                       # :342-360
    n = 50
    failing = random_hosts(n, 10, seed=12, lo=1)
    ref, dev = sims = make(orc, rb, n, 12)
    flags(sims, failing, INGRESS_BLOCKED)
    for _ in range(10):
        assert dev.interval()["event"] == ref.interval()["event"] == "quiet"
    flags(sims, failing, 0)
    while not ref.history:
        ref.interval()
        dev.interval()
    same_run(ref, dev)
    assert dev.history[0]["cut"] == failing and dev.history[0]["path"] == "fast"


def test_edge_failures(orc, rb):
    """the probes of every observer of one live node fail (setEdgeFail on the detector that watches it): it is cut although
    alive, on the device as in simref"""
    n, y = 50, 7
    ref, dev = make(orc, rb, n, 16)
    obs = ref.view.getObserversOf(y)
    assert obs == dev.view.getObserversOf(y)
    for s in (ref, dev):
        for k, o in enumerate(obs):
            s.setEdgeFail(o, k)
    while not ref.history:
        assert ref.interval()["event"] != "stalled" and len(ref.intervals) < 15
        dev.interval()
    same_run(ref, dev)
    assert dev.history[0]["cut"] == [y] and dev.history[0]["path"] == "fast" and dev.history[0]["intervals"] == 11


def test_a_stalling_draw_is_reported(orc, rb):
    n, f, seed = 50, 16, 131
    failing = random_hosts(n, f, seed)
    ref, dev = sims = make(orc, rb, n, seed)
    flags(sims, failing, CRASHED)
    a, b = ref.run(15), dev.run(15)
    assert b["stalled"] and b["stuck"] == a["stuck"] == failing and b["intervals"] == 15
    same_run(ref, dev)


# three of ClusterTest's scenarios at other ring counts and watermarks (the smallest K; K = 11 and 14, where the detector's rows hold a
# hi byte per receiver)
OTHER_KHL = [(3, 3, 1), (11, 10, 4), (14, 12, 5)]


@pytest.mark.parametrize("scenario", ["one-of-five", "failures-of-fifty", "joins-and-fails"])
@pytest.mark.parametrize("K,H,L", OTHER_KHL, ids=["K%d" % k for k, _, _ in OTHER_KHL])
def test_scenarios_at_other_ring_counts(orc, rb, K, H, L, scenario):
    if scenario == "one-of-five":
        n, seed, nj, failing = 5, 1, 0, [2]
    elif scenario == "failures-of-fifty":
        # 12 of 50 as in ClusterTest; at K = 3 with H = 3 that many crashes leave some crashed node without enough live
        # observers to be cut, so 6
        n, seed, nj, failing = 50, 3, 0, random_hosts(50, 12 if K > 3 else 6, 3)
    else:
        n, seed, nj, failing = 30, 13, 10, list(range(2, 7))
    ref, dev = sims = make(orc, rb, n, seed, n_joiners=nj, K=K, H=H, L=L)
    join(sims, range(n, n + nj))
    flags(sims, failing, CRASHED)
    run(sims)
    same_run(ref, dev)
    assert sorted(dev.members()) == sorted([m for m in range(n) if m not in failing] + list(range(n, n + nj)))


# ---- the primitives ------------------------------------------------------------------------------------------------------------
def _view_with_joiners(rb, n, nj, K=10):
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    hosts, ports = W.endpoints(n, nj)
    ids = v.registerJoiners(hosts, ports)
    return v, ids


def test_join_alerts_merge_into_the_interval(rb):
    n, nj, K = 40, 6, 10
    v, jids = _view_with_joiners(rb, n, nj, K)
    exp = v.joinerTables()
    flags = np.zeros(n, np.uint8)
    flags[[3, 17]] = CRASHED
    crashed_obs = int(exp[0][0])
    flags[crashed_obs] = CRASHED                                  # joiner 0 loses (at least) one observer
    fd, plain = rb.EdgeFailureDetectors(v), rb.EdgeFailureDetectors(v)
    for _ in range(11):
        tick = fd.tick(flags, 7)
        assert plain.tick(flags, 7) == tick
    det = fd.alerts()
    assert det                                                    # the crashed nodes' observers notify in this interval
    listed = [jids[4], jids[0], jids[2]]
    na, nc = fd.joinAlerts(listed, 9)
    want = {}
    for o, s, rings in det:
        want.setdefault(o, []).append((o, s, rings))
    for j in listed:
        row = exp[j - n].tolist()
        for o in dict.fromkeys(row):
            if not flags[o] & CRASHED:
                want.setdefault(o, []).append((o, j, [k for k in range(K) if row[k] == o]))
    want = [a for o in sorted(want) for a in want[o]]
    assert fd.alerts() == want and na == len(want)
    src, dst, ring, status, cfg = fd.cells()
    assert nc == len(src) == sum(len(r) for _, _, r in want)
    assert list(zip(src.tolist(), dst.tolist(), ring.tolist())) == [(o, s, r) for o, s, rings in want for r in rings]
    up = dst >= n
    assert (status[up] == 0).all() and (cfg[up] == 9).all() and (status[~up] == 1).all() and (cfg[~up] == 7).all()
    assert not any(o == crashed_obs for o, s, _ in want if s >= n)
    off = fd.senderBatches()
    assert len(off) - 1 == len(np.unique(src)) and all(len(set(src[off[i]: off[i + 1]].tolist())) == 1 for i in range(len(off) - 1))
    # an id that is not a registered joiner: refused, the interval stays as it was
    with pytest.raises(rb.RapidError):
        fd.joinAlerts([jids[1], 5], 9)
    assert fd.alerts() == want
    # one merge per tick: a second call, even with registered joiners only, is refused and leaves the merged interval whole
    with pytest.raises(rb.RapidError, match="already added"):
        fd.joinAlerts([jids[1]], 9)
    assert fd.alerts() == want and fd.n_alerts == na and fd.n_cells == nc
    src2, dst2, ring2, status2, cfg2 = fd.cells()
    assert (status2 == status).all() and (cfg2 == cfg).all() and (dst2 == dst).all()
    # a tick without a join call is today's tick
    assert fd.tick(flags, 7) == plain.tick(flags, 7) and fd.alerts() == plain.alerts()


def test_join_alerts_without_detector_alerts(rb):
    n, nj, K = 200, 3, 10
    v, jids = _view_with_joiners(rb, n, nj, K)
    exp = v.joinerTables()
    fd = rb.EdgeFailureDetectors(v)
    assert fd.tick(np.zeros(n, np.uint8), 1) == (0, 0)
    na, nc = fd.joinAlerts(jids, 1)
    assert na == sum(len(set(r.tolist())) for r in exp) and nc == nj * K
    assert [s for _, s, _ in fd.alerts()] and all(s >= n for _, s, _ in fd.alerts())


def test_find_value(rb):
    R = 1000
    a = rb.PaxosAcceptors(5, R)
    va, vb = (11, 12, 3), (21, 22, 4)
    a.registerFastRoundVotes([700, 40, 41, 999], [va[0], vb[0], va[0], va[0]], [va[2], vb[2], va[2], va[2]], [va[1], vb[1], va[1], va[1]])
    assert a.findValue(va) == 41 and a.findValue(vb) == 40
    assert a.findValue((11, 12, 4)) == -1 and a.findValue((11, 13, 3)) == -1
    assert a.handlePhase1aMessage((2, 9)) == R                   # Phase1a leaves every vval where it was
    assert a.findValue(va) == 41
    vc = (31, 32, 5)
    assert a.findValue(vc) == -1
    assert a.handlePhase2aMessage((2, 9), vc) == R               # Phase2a overwrites them: only then is vc held
    assert a.findValue(vc) == 0 and a.findValue(va) == -1


def test_silent_acceptors(rb):
    R = 300
    silent = np.zeros(R, np.uint8)
    silent[::7] = 1
    a, b = rb.PaxosAcceptors(5, R), rb.PaxosAcceptors(5, R)
    for x in (a, b):
        x.registerFastRoundVotes([1, 7, 8], [5, 5, 5], [2, 2, 2], [6, 6, 6])
    a.setSilent(silent)
    assert a.handlePhase1aMessage((2, 3)) == R - int(silent.sum())
    assert a.handlePhase2aMessage((2, 3), (9, 9, 1)) == R - int(silent.sum())
    for r in (0, 7, 14, 1, 8):
        st = a.read(r)
        if silent[r]:
            assert st == b.read(r)                                # a silent acceptor changed nothing
        else:
            assert st["rnd"] == (2, 3) and st["vval"] == (9, 9, 1)
    a.setSilent(None)                                             # no mask: every acceptor answers, as before
    assert a.handlePhase1aMessage((3, 3)) == R and b.handlePhase1aMessage((3, 3)) == R
    assert b.handlePhase2aMessage((3, 3), (9, 9, 1)) == R


# ---- at scale ------------------------------------------------------------------------------------------------------------------
def test_ten_thousand_nodes_against_simref(orc, rb):
    n = 10_000
    crashed = W.pick_smallest(n, n // 100, 21).tolist()
    ref, dev = sims = make(orc, rb, n, 21)
    flags(sims, crashed, CRASHED)
    run(sims, 15)
    same_run(ref, dev)


def _no_dark_draw(obs, n, frac, seed, L=4):
    """a crash set of frac * n in which every crashed node keeps at least L live observers, so every crashed node reaches the
    proposal (a node reported by fewer than L observers cannot be added by invalidation and can block the cut)"""
    K = obs.shape[1]
    order = np.argsort(W.splitmix64(np.arange(n, dtype=np.uint64) ^ np.uint64(seed)), kind="stable")
    subj = [[] for _ in range(n)]
    for y in range(n):
        for o in obs[y]:
            subj[o].append(y)
    down = np.zeros(n, np.int32)                                  # crashed observers per node
    out = np.zeros(n, bool)
    want, got = int(frac * n), 0
    for x in order.tolist():
        if got == want:
            break
        if down[x] > K - L or any(down[y] >= K - L for y in subj[x]):
            continue
        out[x] = True
        got += 1
        for y in subj[x]:
            down[y] += 1
    return np.nonzero(out)[0].tolist()


def test_hundred_thousand_nodes_churn(rb):
    n, nj = 100_000, 200
    crashed = W.pick_smallest(n, n // 100, 22).tolist()
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=22)
    join((s,), range(n, n + nj))
    flags((s,), crashed, CRASHED)
    out = s.run(15)
    assert out["converged"]
    assert sorted(s.members()) == sorted(set(range(n)) - set(crashed) | set(range(n, n + nj)))
    assert sorted(t for h in s.history for t in h["cut"]) == sorted(crashed + list(range(n, n + nj)))
    print("1e5 churn:", [{k: h[k] for k in ("path", "intervals", "size", "detect_ms", "view_change_ms", "handles_ms")} for h in s.history])


def test_ten_thousand_nodes_thirty_percent_crashed(rb):
    """0.7 N voters < the fast quorum N - floor((N-1)/4): the classic round decides, the crashed acceptors silent.

    Run at 10^4 nodes rather than 10^5: at 10^5 the alerting interval holds about 2 * 10^5 alerts from about 7 * 10^4 senders,
    handled as one sequence of per-sender batches, and one run takes longer than a test may (DESIGN.md §4.11, open questions)."""
    n = 10_000
    v = rb.MembershipView.from_packed(10, *W.packed_endpoints(0, n))
    obs, _ = v.tables()
    v.close()
    crashed = _no_dark_draw(obs, n, 0.30, 23)
    assert len(crashed) == 3_000
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=23)
    flags((s,), crashed, CRASHED)
    out = s.run(15)
    assert out["converged"] and sorted(s.members()) == sorted(set(range(n)) - set(crashed))
    h = s.history
    # a receiver may announce part of the crashed set before the rest of the senders' batches reach it, so the first cut can
    # leave some crashed nodes for a later configuration
    assert h[0]["path"] == "classic" and h[0]["intervals"] == 12                 # proposals in interval 10, the fallback in 11
    assert h[0]["announced"] == h[0]["votes"] == n - len(crashed)
    assert sorted(t for c in h for t in c["cut"]) == crashed


def test_one_million_nodes_one_percent_crashed(rb):
    """the Fig. 8 shape at 10^6: one fast-path view change whose cut is the crashed set"""
    n = 1_000_000
    crashed = W.pick_smallest(n, n // 100, 24).tolist()
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=24)
    flags((s,), crashed, CRASHED)
    out = s.run(15)
    assert out["converged"] and len(s.history) == 1
    h = s.history[0]
    assert h["path"] == "fast" and h["cut"] == crashed and h["size"] == n - len(crashed) and h["intervals"] == 11
    assert [r["event"] for r in s.intervals] == ["quiet"] * 10 + ["decided-fast"]
