"""ClusterTest's leave and rejoin scenarios (ClusterTest.java:417-521) written once for the reference of tests/simref.py alone
(test_oracle_cluster_leave_rejoin.py) or in lockstep with the device's ClusterSimulation (test_gpu_cluster_leave_rejoin.py),
through simref's harness.  Every step is applied to every simulation; the scenario's own assertions are made on the first one,
and the callers compare the runs.  NOT a pytest module."""
from simref import CRASHED, flags, join, leave, make, random_hosts, rejoin, run, steps
from rapid_b200 import workloads as W


def fresh_id(k):
    """a NodeId no scenario gives at creation or to a first join (those are W.node_ids of the tag)"""
    hi, lo = W.node_ids((1 << 40) + k, 1)
    return int(hi[0]), int(lo[0])


# ---- the scenarios ---------------------------------------------------------------------------------------------------------------
def leaving(orc, rb, seed=31):
    """testLeaving (:509-521): a cluster grown by single joins from 2 to 11 members; member 0 leaves, the other 10 agree on the
    cut [0], decided in the leave's interval"""
    sims = make(orc, rb, 2, seed, n_joiners=9)
    for t in range(2, 11):
        join(sims, [t])
        run(sims)
        assert sorted(sims[0].members()) == list(range(t + 1))
    before = len(sims[0].history)
    leave(sims, [0])
    run(sims)
    h = sims[0].history[before:]
    assert [c["cut"] for c in h] == [[0]] and h[0]["intervals"] == 1 and h[0]["path"] == "fast"
    assert sorted(sims[0].members()) == list(range(1, 11))
    return sims


def rejoin_single_node(orc, rb, tag=3, seed=32):
    """testRejoinSingleNode (:417-445): of 10, one node crashes; once it is cut it rejoins with a new NodeId.  Twice."""
    sims = make(orc, rb, 10, seed)
    for rnd in range(2):
        flags(sims, [tag], CRASHED)
        run(sims)
        assert tag not in sims[0].members() and sims[0].history[-1]["cut"] == [tag]
        rejoin(sims, tag, fresh_id(rnd))
        run(sims)
        assert sorted(sims[0].members()) == list(range(10)) and sims[0].history[-1]["cut"] == [tag]
    return sims


def rejoin_same_configuration(orc, rb, tag=6, seed=33, refuse=True):
    """testRejoinSingleNodeSameConfiguration (:447-472): while the crashed incarnation is still a member, a rejoin is refused
    (HOSTNAME_ALREADY_IN_RING) and changes nothing; after the detectors cut it, the same rejoin succeeds"""
    sims = make(orc, rb, 10, seed)
    flags(sims, [tag], CRASHED)
    steps(sims, 4)
    refused = 0
    if refuse:
        for s in sims:
            try:
                s.rejoin(tag, *fresh_id(7))
            except ValueError:
                refused += 1
        assert refused == len(sims)
    run(sims)
    assert sims[0].history[-1]["cut"] == [tag] and sims[0].history[-1]["intervals"] == 11
    rejoin(sims, tag, fresh_id(7))
    run(sims)
    assert sorted(sims[0].members()) == list(range(10))
    return sims


def rejoin_multiple_nodes(orc, rb, mode, seed=34):
    """testRejoinMultipleNodes (:474-505): of 30, five nodes go (crash or graceful leave) and rejoin with new NodeIds, three
    rounds; the cluster is whole after every round"""
    n = 30
    sims = make(orc, rb, n, seed)
    for rnd in range(3):
        gone = random_hosts(n, 5, seed * 10 + rnd)
        if mode == "crash":
            flags(sims, gone, CRASHED)
        else:
            leave(sims, gone)
        run(sims, 40)
        assert sorted(sims[0].members()) == [t for t in range(n) if t not in gone]
        for j, t in enumerate(gone):
            rejoin(sims, t, fresh_id(100 * rnd + j))
        run(sims, 40)
        assert sorted(sims[0].members()) == list(range(n))
    return sims


def leave_against_crash(orc, rb, how, n=50, tag=17, seed=35):
    """the same draw, one node going two ways: a graceful leave is decided in interval 0, a crash in interval 10"""
    sims = make(orc, rb, n, seed)
    if how == "leave":
        leave(sims, [tag])
    else:
        flags(sims, [tag], CRASHED)
    run(sims)
    h = sims[0].history
    assert len(h) == 1 and h[0]["cut"] == [tag] and h[0]["path"] == "fast"
    assert h[0]["intervals"] == (1 if how == "leave" else 11)
    return sims


def adjacent_pair(view, n, start):
    """(observer, subject) with both members: the first member from start that observes another"""
    for y in range(start, n):
        o = view.getObserversOf(y)[0]
        if o != y:
            return o, y
    raise AssertionError("no pair")


def adjacent_leavers(orc, rb, n=50, seed=36):
    """two leavers, one observing the other: the observed one loses that observer's LeaveMessages (it has shut down too).
    Whatever the implicit reports of invalidateFailingEdges make of it, both end up cut."""
    sims = make(orc, rb, n, seed)
    o, y = adjacent_pair(sims[0].view, n, 5)
    leave(sims, [y, o])
    run(sims)
    assert sorted(sims[0].members()) == [t for t in range(n) if t not in (o, y)]
    return sims


def leaver_with_crashed_observers(orc, rb, n=100, tag=40, seed=37):
    """every observer of the leaver crashes in the leave's interval: its leave raises nothing, the observers are cut, and the
    next configuration's detectors cut the leaver"""
    sims = make(orc, rb, n, seed)
    obs = sorted(set(sims[0].view.getObserversOf(tag)))
    flags(sims, obs, CRASHED)
    leave(sims, [tag])
    r = steps(sims, 1)[0]
    assert r["leavers"] == 1 and r["alerts"] == 0
    run(sims)
    h = sims[0].history
    assert sorted(t for c in h[:-1] for t in c["cut"]) == obs
    assert h[-1]["cut"] == [tag] and h[-1]["intervals"] == 11
    assert sorted(sims[0].members()) == [t for t in range(n) if t not in obs and t != tag]
    return sims


def refused(sims, call):
    """call(s) raises ValueError on every simulation"""
    for s in sims:
        try:
            call(s)
        except ValueError:
            continue
        raise AssertionError("accepted")


def refusals(orc, rb, seed=38, refuse=True):
    """refused leaves and rejoins raise ValueError and change nothing (the caller compares with refuse=False); a rejoin with any
    NodeId this simulation was given is refused, with a new one it is admitted"""
    n = 12
    sims = make(orc, rb, n, seed, n_joiners=1)
    join(sims, [n])
    flags(sims, [4], CRASHED)
    hi, lo = W.node_ids(0, n + 1)
    if refuse:
        for bad in ([4], [99], [n], [2, 2], [3, 4]):                             # crashed, unknown, pending joiner, twice, mixed
            refused(sims, lambda s: s.leave(bad))
        for tag, nid in ((5, fresh_id(1)), (4, fresh_id(1)),                      # members (the second one crashed)
                         (n, fresh_id(2))):                                       # pending
            refused(sims, lambda s: s.rejoin(tag, *nid))
    run(sims)
    assert sorted(sims[0].members()) == [t for t in range(n + 1) if t != 4]
    if refuse:
        for j in (n, 4, 9):                                                       # a joiner's, its own old one, a member's
            nid = (int(hi[j]), int(lo[j]))
            refused(sims, lambda s: s.rejoin(4, *nid))
        refused(sims, lambda s: s.leave([4]))                                     # not a member any more
    rejoin(sims, 4, fresh_id(3))
    run(sims)
    assert sorted(sims[0].members()) == list(range(n + 1))
    return sims
