"""Graceful leaves and rejoins on the device: rapid_fdet_merge_alerts (join and leave alerts merged into the failure-detector
interval) on its own against the device view's getObserversOf / getRingNumbers; ClusterSimulation.leave / rejoin against
tests/simref.py interval by interval and configuration by configuration on ClusterTest's leave and rejoin scenarios
(leave_scenarios.py) and at 10^4 nodes; and, checked on their outcome, 1 % leaving at 10^6 nodes and rolling restarts at 10^5."""
import numpy as np
import pytest

import leave_scenarios as S
from simref import CRASHED, flags, leave, make, rejoin, run, same_run
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


# ---- the merge on its own ------------------------------------------------------------------------------------------------------
def _view(rb, n, nj=0, K=10):
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    jids = v.registerJoiners(*W.endpoints(n, nj)) if nj else []
    return v, jids


def leave_alerts(v, flags, leavers, K=10):
    """[(sender, subject, rings)] of the listed leavers, in list order then k, from the view's own queries"""
    out = []
    for l in leavers:
        for o in v.getObserversOf(l):
            if not flags[o] & CRASHED:
                out.append((o, l, v.getRingNumbers(o, l)))
    return out


def join_alerts(exp, n, flags, joiners, K=10):
    out = []
    for j in joiners:
        row = exp[j - n].tolist()
        for o in dict.fromkeys(row):
            if not flags[o] & CRASHED:
                out.append((o, j, [k for k in range(K) if row[k] == o]))
    return out


def by_sender(*groups):
    """per sender in ascending id, the groups' alerts in group order (each group already in its own order)"""
    want = {}
    for g in groups:
        for a in g:
            want.setdefault(a[0], []).append(a)
    return [a for o in sorted(want) for a in want[o]]


def test_leave_alerts_are_the_observer_rows(rb):
    n, K = 12, 10
    v, _ = _view(rb, n)
    a, b = 3, 8                                                   # a's observers live but one, b crashed itself
    obs_a = v.getObserversOf(a)
    dead = obs_a[0]
    assert dead not in v.getObserversOf(b) and b not in obs_a
    flags = np.zeros(n, np.uint8)
    flags[[dead, b]] = CRASHED
    fd = rb.EdgeFailureDetectors(v)
    assert fd.tick(flags, 7) == (0, 0)
    na, nc = fd.mergeAlerts([], [a, b], 9)
    want = by_sender(leave_alerts(v, flags, [a, b]))
    assert fd.alerts() == want and na == len(want)
    per = {l: [x for x in want if x[1] == l] for l in (a, b)}
    assert len(per[a]) == K - obs_a.count(dead)                  # one alert per live entry of getObserversOf, repeats kept
    assert len(per[b]) == K and b not in [x[0] for x in want]    # a crashed leaver is still announced; it sends nothing
    assert dead not in [x[0] for x in want]
    mult = {o: v.getObserversOf(b).count(o) for o in set(v.getObserversOf(b))}
    assert max(mult.values()) > 1                                # some observer repeats on this view
    assert sum(len(r) for _, s, r in want if s == b) == sum(m * m for m in mult.values())
    src, dst, ring, status, cfg = fd.cells()
    assert nc == len(src) == sum(len(r) for _, _, r in want)
    assert list(zip(src.tolist(), dst.tolist(), ring.tolist())) == [(o, s, r) for o, s, rings in want for r in rings]
    assert (status == 1).all() and (cfg == 9).all()


def test_tick_join_and_leave_alerts_in_one_interval(rb):
    n, nj, K = 14, 3, 10
    v, jids = _view(rb, n, nj, K)
    exp = v.joinerTables()
    flags = np.zeros(n, np.uint8)
    flags[[2, 9]] = CRASHED
    fd = rb.EdgeFailureDetectors(v)
    for _ in range(11):
        fd.tick(flags, 7)
    det = fd.alerts()
    assert det
    joiners, leavers = [jids[2], jids[0]], [5, 11]
    na, nc = fd.mergeAlerts(joiners, leavers, 9)
    want = by_sender(det, join_alerts(exp, n, flags, joiners, K), leave_alerts(v, flags, leavers))
    got = fd.alerts()
    assert got == want and na == len(want)
    kinds = {}
    for o, s, _ in got:
        kinds.setdefault(o, []).append("tick" if (o, s) in {(x[0], x[1]) for x in det} else ("join" if s >= n else "leave"))
    assert any(k[0] == "tick" and "join" in k and k[-1] == "leave" for k in kinds.values())    # a sender with all three
    for k in kinds.values():
        assert k == sorted(k, key=["tick", "join", "leave"].index)
    src, dst, ring, status, cfg = fd.cells()
    assert nc == len(src)
    up, tick = dst >= n, cfg == 7
    assert (status[up] == 0).all() and (cfg[up] == 9).all()
    assert (status[~up] == 1).all() and int(tick.sum()) == sum(len(r) for _, _, r in det)
    off = fd.senderBatches()
    assert len(off) - 1 == len(np.unique(src))


def test_two_member_view(rb):
    v, _ = _view(rb, 2)
    fd = rb.EdgeFailureDetectors(v)
    fd.tick(np.zeros(2, np.uint8), 1)
    na, nc = fd.mergeAlerts([], [0], 1)
    assert (na, nc) == (10, 100) and fd.alerts() == [(1, 0, list(range(10)))] * 10
    one, _ = _view(rb, 1)
    fd1 = rb.EdgeFailureDetectors(one)
    fd1.tick(np.zeros(1, np.uint8), 1)
    assert fd1.mergeAlerts([], [0], 1) == (0, 0)                 # getObserversOf is empty in a one-member view


def test_refusals_leave_the_interval_unchanged(rb):
    n, nj = 30, 2
    v, jids = _view(rb, n, nj)
    flags = np.zeros(n, np.uint8)
    flags[[4, 19]] = CRASHED
    fd = rb.EdgeFailureDetectors(v)
    with pytest.raises(rb.RapidError):
        fd.mergeAlerts([], [1], 3)                                # no tick yet
    for _ in range(11):
        fd.tick(flags, 3)
    before = (fd.alerts(), [a.copy() for a in fd.cells()], fd.n_alerts, fd.n_cells)
    for j, l in (([], [jids[0]]), ([], [-1]), ([], [n + nj]), ([5], []), ([jids[0]], [2, n])):
        with pytest.raises(rb.RapidError):
            fd.mergeAlerts(j, l, 3)
    after = (fd.alerts(), fd.cells(), fd.n_alerts, fd.n_cells)
    assert after[0] == before[0] and after[2:] == before[2:]
    assert all((x == y).all() and x.dtype == y.dtype for x, y in zip(after[1], before[1]))
    na, nc = fd.mergeAlerts([jids[1]], [7], 3)
    merged = (fd.alerts(), [a.copy() for a in fd.cells()])
    for j, l in (([], [8]), ([jids[0]], []), ([], [])):
        with pytest.raises(rb.RapidError, match="already added"):
            fd.mergeAlerts(j, l, 3)
    with pytest.raises(rb.RapidError, match="already added"):
        fd.joinAlerts([jids[0]], 3)
    assert fd.alerts() == merged[0] and all((x == y).all() for x, y in zip(fd.cells(), merged[1]))
    assert (fd.n_alerts, fd.n_cells) == (na, nc)
    w, _ = _view(rb, 20)                                          # the view changed since the tick
    fw = rb.EdgeFailureDetectors(w)
    fw.tick(np.zeros(20, np.uint8), 1)
    w.applyCut([3])
    with pytest.raises(rb.RapidError, match="view changed"):
        fw.mergeAlerts([], [1], 1)


def test_join_alerts_is_the_merge_without_leavers(rb):
    n, nj = 60, 4
    v, jids = _view(rb, n, nj)
    flags = np.zeros(n, np.uint8)
    flags[[1, 22, 40]] = CRASHED
    a, b = rb.EdgeFailureDetectors(v), rb.EdgeFailureDetectors(v)
    for _ in range(11):
        assert a.tick(flags, 5) == b.tick(flags, 5)
    assert a.joinAlerts([jids[3], jids[1]], 6) == b.mergeAlerts([jids[3], jids[1]], [], 6)
    assert a.alerts() == b.alerts()
    assert all((x == y).all() for x, y in zip(a.cells(), b.cells()))
    assert (a.senderBatches() == b.senderBatches()).all()


# ---- the driver against simref -----------------------------------------------------------------------------------------------------
def test_leaving(orc, rb):
    ref, dev = S.leaving(orc, rb)
    same_run(ref, dev)


def test_rejoin_single_node(orc, rb):
    ref, dev = S.rejoin_single_node(orc, rb)
    same_run(ref, dev)


def test_rejoin_single_node_same_configuration(orc, rb):
    ref, dev = S.rejoin_same_configuration(orc, rb)
    same_run(ref, dev)


@pytest.mark.parametrize("mode", ["crash", "leave"])
def test_rejoin_multiple_nodes(orc, rb, mode):
    ref, dev = S.rejoin_multiple_nodes(orc, rb, mode)
    same_run(ref, dev)


@pytest.mark.parametrize("how", ["leave", "crash"])
def test_leave_against_crash_on_the_same_draw(orc, rb, how):
    ref, dev = S.leave_against_crash(orc, rb, how)
    same_run(ref, dev)


def test_adjacent_leavers(orc, rb):
    ref, dev = S.adjacent_leavers(orc, rb)
    same_run(ref, dev)


def test_leaver_whose_observers_crashed(orc, rb):
    ref, dev = S.leaver_with_crashed_observers(orc, rb)
    same_run(ref, dev)


def test_refusals(orc, rb):
    ref, dev = S.refusals(orc, rb)
    same_run(ref, dev)


def test_ten_thousand_nodes_leaves_rejoins_and_crashes(orc, rb):
    n = 10_000
    sims = make(orc, rb, n, 41)
    drawn = W.pick_smallest(n, n // 100, 41).tolist()
    gone, crashed = drawn[::2], drawn[1::2]
    flags(sims, crashed, CRASHED)
    leave(sims, gone)
    run(sims, 15)
    assert sorted(sims[1].members()) == sorted(set(range(n)) - set(drawn))
    for j, t in enumerate(drawn):
        rejoin(sims, t, S.fresh_id(j))
    run(sims, 15)
    assert sorted(sims[1].members()) == list(range(n))
    same_run(*sims)


@pytest.mark.parametrize("K,H,L", [(3, 3, 1), (11, 10, 4), (14, 12, 5)], ids=["K3", "K11", "K14"])
def test_leave_and_rejoin_wave_at_other_ring_counts(orc, rb, K, H, L):
    """a wave of graceful leaves and a crash, then every one of them rejoins with a new NodeId, at other ring counts and
    watermarks"""
    n = 40
    sims = make(orc, rb, n, 44, K=K, H=H, L=L)
    gone, crashed = [3, 17, 29], [11]
    leave(sims, gone)
    flags(sims, crashed, CRASHED)
    run(sims)
    assert sorted(sims[1].members()) == [t for t in range(n) if t not in gone + crashed]
    for j, t in enumerate(gone + crashed):
        rejoin(sims, t, S.fresh_id(200 + j))
    run(sims)
    assert sorted(sims[1].members()) == list(range(n))
    same_run(*sims)


# ---- at scale ----------------------------------------------------------------------------------------------------------------------
def apart(rb, n, count, seed):
    """count members, in pick_smallest order of the seed, none of which observes another"""
    v = rb.MembershipView.from_packed(10, *W.packed_endpoints(0, n))
    obs, subj = v.tables()
    v.close()
    chosen = np.zeros(n, bool)
    order = np.argsort(W.splitmix64(np.arange(n, dtype=np.uint64) ^ np.uint64(seed)), kind="stable")
    got = 0
    for x in order.tolist():
        if got == count:
            break
        if chosen[obs[x]].any() or chosen[subj[x]].any():
            continue
        chosen[x] = True
        got += 1
    return np.nonzero(chosen)[0].tolist()


def test_one_million_nodes_one_percent_leave(rb):
    n = 1_000_000
    leavers = apart(rb, n, n // 100, 42)
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=42)
    s.leave(leavers)
    out = s.run(15)
    assert out["converged"]
    h = s.history
    assert h[0]["path"] == "fast" and h[0]["intervals"] == 1 and s.intervals[0]["event"] == "decided-fast"
    assert s.intervals[0]["leavers"] == len(leavers) and s.intervals[0]["alerts"] == 10 * len(leavers)
    assert sorted(t for c in h for t in c["cut"]) == leavers and h[-1]["size"] == n - len(leavers)
    print("1e6 leave:", [{k: c[k] for k in ("path", "intervals", "size", "detect_ms", "view_change_ms", "handles_ms")} for c in h],
          "alerting interval device ms:", s.intervals[0]["device_ms"])
    s.close()


def test_hundred_thousand_nodes_rolling_restart(rb):
    """three disjoint waves of 1 % leave and come back with new NodeIds.  A wave may hold a leaver that observes another;
    the implicit reports of invalidateFailingEdges then complete the cut, and if a draw split it over two configurations the
    union would still be the wave, which is what is asserted."""
    n, w = 100_000, 1_000
    drawn = W.pick_smallest(n, 3 * w, 43).tolist()
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=43)
    first = s.cfg
    for k in range(3):
        wave = drawn[k::3]
        mark = len(s.history)
        s.leave(wave)
        assert s.run(15)["converged"]
        assert sorted(t for c in s.history[mark:] for t in c["cut"]) == wave
        mark = len(s.history)
        for j, t in enumerate(wave):
            s.rejoin(t, *S.fresh_id(k * w + j))
        assert s.run(15)["converged"]
        assert sorted(t for c in s.history[mark:] for t in c["cut"]) == wave
        assert sorted(s.members()) == list(range(n))
    assert all(c["path"] == "fast" for c in s.history) and s.cfg != first
    print("1e5 rolling:", [{k: c[k] for k in ("path", "intervals", "size", "detect_ms", "view_change_ms", "handles_ms")}
                           for c in s.history])
    s.close()
