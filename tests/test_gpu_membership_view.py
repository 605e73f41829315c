"""GPU MembershipView (librapid_b200) vs the oracle, through the C ABI: ring order, keys, observer / subject /
expected-observer tables, ring numbers, configuration id; plus the structural invariants MembershipViewTest asserts
(rapid/src/test/java/com/vrg/rapid/MembershipViewTest.java)."""
import numpy as np
import pytest

from helpers import OracleWorld
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu
K = 10


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.mark.parametrize("n", [1, 2, 3, 50, 1000, 5000])
def test_rings_tables_config_id_match_oracle(orc, rb, n):
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    assert v.getMembershipSize() == n
    for k in range(K):
        np.testing.assert_array_equal(v.getRing(k), np.asarray(w.view.getRing(k), np.int32))
        keys = v.keys(k)
        for i in (0, n // 2, n - 1):
            assert int(keys[i]) == w.view.key(k, i)
    obs, subj = v.tables()
    if n > 1:
        o_obs, o_subj = w.tables()
        np.testing.assert_array_equal(obs, o_obs)
        np.testing.assert_array_equal(subj, o_subj)
    for i in {0, n // 3, n - 1}:
        assert v.getObserversOf(i) == w.view.getObserversOf(i)          # [] when n == 1
        assert v.getSubjectsOf(i) == w.view.getSubjectsOf(i)
    assert v.getCurrentConfigurationId(w.id_high, w.id_low) == w.view.getCurrentConfigurationId()
    # identifiers of departed nodes stay in identifiersSeen (MembershipView.java:167-201): more ids than members
    hi2, lo2 = W.node_ids(0, n + 7)
    ref = orc.MembershipView(w.u, K, np.arange(n, dtype=np.int32), hi2, lo2)
    assert v.getCurrentConfigurationId(hi2, lo2) == ref.getCurrentConfigurationId()


def test_not_in_ring_and_small_views(rb):
    v = rb.MembershipView(K, ["127.0.0.1"], [1])
    assert v.getObserversOf(0) == [] and v.getSubjectsOf(0) == []       # MembershipViewTest.java:166-176
    with pytest.raises(rb.NodeNotInRingException):
        v.getObserversOf(1)
    with pytest.raises(rb.NodeNotInRingException):
        v.getSubjectsOf(5)
    assert v.getExpectedObserversOf("127.0.0.1", 2) == [0] * K          # :298-313
    v2 = rb.MembershipView(K, ["127.0.0.1", "127.0.0.1"], [1, 2])
    assert v2.getObserversOf(0) == [1] * K and v2.getSubjectsOf(0) == [1] * K   # :221-235
    empty = rb.MembershipView(K)
    assert empty.getMembershipSize() == 0
    assert empty.getExpectedObserversOf("127.0.0.1", 1) == []
    with pytest.raises(rb.NodeNotInRingException):
        empty.getObserversOf(0)


def test_duplicate_endpoint_rejected(rb):
    with pytest.raises(rb.NodeAlreadyInRingException):
        rb.MembershipView(K, ["a", "b", "a"], [1, 1, 1])


def test_k_observers_and_subjects_for_every_node(rb):                  # MembershipViewTest.java:268-293
    hosts, ports = ["127.0.0.1"] * 1000, list(range(1000))
    v = rb.MembershipView(K, hosts, ports)
    obs, subj = v.tables()
    assert obs.shape == (1000, K) and (obs >= 0).all() and (subj >= 0).all()
    assert (obs != np.arange(1000)[:, None]).all()
    # observer/subject are inverse relations on every ring
    for k in range(K):
        assert (subj[obs[:, k], k] == np.arange(1000)).all()


def test_expected_observers_and_ring_numbers(orc, rb):
    n, nj = 400, 25
    w = OracleWorld(orc, n, K, n_joiners=nj)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    hosts, ports = w.joiner_endpoints()
    for j in range(nj):
        assert v.getExpectedObserversOf(hosts[j], int(ports[j])) == w.view.getExpectedObserversOf(n + j)
    ids = v.registerJoiners(hosts, ports)
    assert ids == list(range(n, n + nj)) and v.numJoiners() == nj
    for k in (0, 9):
        keys = v.keys(k)
        for j in (0, nj - 1):
            assert int(keys[n + j]) == w.view.key(k, n + j)
    with pytest.raises(rb.NodeAlreadyInRingException):
        h0, p0 = W.endpoints(5, 1)
        v.registerJoiners(h0, p0)
    for i in range(0, n, 37):
        for o in set(w.view.getObserversOf(i)):
            assert v.getRingNumbers(o, i) == w.view.getRingNumbers(o, i)
    # expected observers of a member-shaped endpoint that is already in the ring: still predecessors
    assert v.getExpectedObserversOf(*[x[0] for x in W.endpoints(7, 1)][:1], int(W.endpoints(7, 1)[1][0])) == w.view.getExpectedObserversOf(7)


def test_long_hostnames(orc, rb):
    """XXH64's >= 32-byte stripe loop on the device"""
    hosts = ["node-%04d.some-very-long-datacenter-name.example.internal" % i for i in range(64)]
    ports = [9000 + (i % 3) for i in range(64)]
    u = orc.Universe()
    tags = [u.add(h, p) for h, p in zip(hosts, ports)]
    ref = orc.MembershipView(u, K, tags, [], [])
    v = rb.MembershipView(K, hosts, ports)
    for k in range(K):
        assert v.getRing(k).tolist() == ref.getRing(k)
    assert v.getCurrentConfigurationId([], []) == ref.getCurrentConfigurationId()


def test_apply_cut_matches_ring_delete_and_add(orc, rb):
    """decideViewChange on the device view == ringDelete / ringAdd on the oracle view (MembershipService.java:385-444)"""
    n, nj = 300, 12
    w = OracleWorld(orc, n, K, n_joiners=nj)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    v.registerJoiners(*w.joiner_endpoints())
    rng = np.random.default_rng(8)
    leave = sorted(rng.choice(n, size=9, replace=False).tolist())
    join = [n + j for j in sorted(rng.choice(nj, size=5, replace=False).tolist())]
    mapping = v.applyCut(leave + join)
    # the same decision applied to the oracle view
    hi, lo = W.node_ids(n, nj)
    for x in leave:
        w.view.ringDelete(x)
    for x in join:
        w.view.ringAdd(x, (int(hi[x - n]), int(lo[x - n])))
    assert v.getMembershipSize() == w.view.getMembershipSize() == n - 9 + 5
    inv = {int(new): old for old, new in enumerate(mapping.tolist()) if new >= 0}
    for k in range(K):
        assert [inv[i] for i in v.getRing(k).tolist()] == w.view.getRing(k)
    for old in (0, 17, join[0]):
        if mapping[old] >= 0:
            assert [inv[i] for i in v.getObserversOf(int(mapping[old]))] == w.view.getObserversOf(old)
            assert [inv[i] for i in v.getSubjectsOf(int(mapping[old]))] == w.view.getSubjectsOf(old)
    assert all(mapping[x] == -1 for x in leave) and all(mapping[x] >= 0 for x in join)
    # identifiersSeen keeps the ids of the departed (MembershipView.java:167-201): same configuration id
    ids_hi = np.concatenate([w.id_high, hi[[x - n for x in join]]])
    ids_lo = np.concatenate([w.id_low, lo[[x - n for x in join]]])
    assert v.getCurrentConfigurationId(ids_hi, ids_lo) == w.view.getCurrentConfigurationId()
    with pytest.raises(rb.RapidError):
        v.applyCut([0, 0])
    # a detector on the new view works
    cl = rb.VirtualCluster(v, 9, 4)
    obs, _ = v.tables()
    b = W.c2_simultaneous_crash(obs, v.n, 0.01)
    res = cl.handleBatch(5, b.src, b.dst, b.ring, b.status)
    assert set(res.proposal_len.tolist()) == {len(b.expected_cut)}


def test_apply_cut_with_node_ids_uuid_rule_and_device_config_id(orc, rb):
    """identifiersSeen lives on the device: an admitted joiner's NodeId joins it, the ids of the departed stay
    (MembershipView.java:167-201), a NodeId seen before is refused (UUIDAlreadySeenException, :126-128) and leaves the view
    untouched; getCurrentConfigurationId comes from that set without the caller handing identifiers in."""
    n, nj = 700, 40
    w = OracleWorld(orc, n, K, n_joiners=nj)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    v.setNodeIds(w.id_high, w.id_low)
    assert v.currentConfigurationId() == w.view.getCurrentConfigurationId()
    first = v.registerJoiners(*w.joiner_endpoints())[0]
    hi, lo = W.node_ids(n, nj)
    v.setJoinerIds(first, hi, lo)
    rng = np.random.default_rng(21)
    ever = set()                                          # joiners admitted at some point: their NodeIds are used up
    for round_ in range(3):
        members = v.getMembershipSize()
        tot = members + v.numJoiners()
        # ids are renumbered after every cut: keep the oracle's tags alongside
        if round_ == 0:
            tag_of = list(range(n + nj))                    # device id -> oracle tag
        leave = sorted(rng.choice(members, size=11, replace=False).tolist())
        joiners = list(range(members, tot))
        join = sorted(rng.choice(joiners, size=min(6, len(joiners)), replace=False).tolist()) if joiners else []
        mapping = v.applyCut(leave + join)
        for x in leave:
            w.view.ringDelete(tag_of[x])
        for x in join:
            t = tag_of[x]
            w.view.ringAdd(t, (int(hi[t - n]), int(lo[t - n])))
            ever.add(t)
        new_tag = [None] * v.getMembershipSize()
        for old, new in enumerate(mapping.tolist()):
            if new >= 0:
                new_tag[new] = tag_of[old]
        tag_of = new_tag
        assert v.getMembershipSize() == w.view.getMembershipSize()
        for k in range(K):
            assert [tag_of[i] for i in v.getRing(k).tolist()] == w.view.getRing(k)
        assert v.currentConfigurationId() == w.view.getCurrentConfigurationId()
        # joiners that were not admitted are dropped: register the rest again for the next round
        rest = [t for t in range(n, n + nj) if t not in tag_of and t not in ever]
        if rest and round_ < 2:
            hosts, ports = W.endpoints(n, nj)
            sel = [t - n for t in rest]
            first = v.registerJoiners([hosts[i] for i in sel], [ports[i] for i in sel])[0]
            v.setJoinerIds(first, hi[sel], lo[sel])
            tag_of = tag_of + rest
    # UUIDAlreadySeenException: a new endpoint that re-uses the NodeId of a node that LEFT (its id is still in identifiersSeen)
    before = (v.getMembershipSize(), v.getRing(0).tolist(), v.currentConfigurationId())
    hosts, ports = W.endpoints(n + nj, 1)
    jid = v.registerJoiners(hosts, ports)[0]
    v.setJoinerIds(jid, [int(w.id_high[5])], [int(w.id_low[5])])
    with pytest.raises(rb.UUIDAlreadySeenException):
        v.applyCut([jid])
    assert (v.getMembershipSize(), v.getRing(0).tolist(), v.currentConfigurationId()) == before
    # two members with the same NodeId are refused up front
    v2 = rb.MembershipView.from_packed(K, *w.member_packed())
    bad_hi = w.id_high.copy(); bad_lo = w.id_low.copy()
    bad_hi[3], bad_lo[3] = bad_hi[9], bad_lo[9]
    with pytest.raises(rb.UUIDAlreadySeenException):
        v2.setNodeIds(bad_hi, bad_lo)


@pytest.mark.parametrize("n", [1, 2, 4095, 4096, 4097, 20_000])
def test_rings_from_the_hand_written_radix_sort(orc, rb, n):
    """ring order = signed 64-bit key order, sizes around the sort's 4096-pair tile and several tiles"""
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    for k in (0, K - 1):
        ring = v.getRing(k)
        keys = v.keys(k)[ring]
        assert (np.diff(keys) > 0).all() and sorted(ring.tolist()) == list(range(n))
        assert ring.tolist() == w.view.getRing(k)


def test_apply_cut_at_scale_stays_on_the_device(rb):
    """1 % churn of a 200,000-node view: 1,000 leave, 1,000 join; rings stay sorted, ids stay dense, tables consistent"""
    n, nj = 200_000, 1000
    hb, off, ports = W.packed_endpoints(0, n + nj)
    v = rb.MembershipView.from_packed(K, hb[: off[n]], off[: n + 1], ports[:n])
    hosts, jports = W.endpoints(n, nj)
    v.registerJoiners(hosts, jports)
    keys_before = {k: v.keys(k).copy() for k in (0, 3)}
    rng = np.random.default_rng(5)
    leave = np.sort(rng.choice(n, size=1000, replace=False))
    mapping = v.applyCut(np.concatenate([leave, np.arange(n, n + nj)]).astype(np.int32))
    assert v.getMembershipSize() == n and v.numJoiners() == 0
    assert (mapping[leave] == -1).all() and (np.sort(mapping[mapping >= 0]) == np.arange(n)).all()
    inv = np.empty(n, np.int64); old = np.nonzero(mapping >= 0)[0]; inv[mapping[old]] = old
    for k in (0, 3):
        ring = v.getRing(k)
        kk = v.keys(k)
        assert (np.diff(kk[ring]) > 0).all()
        # every surviving node kept its key under its new id
        assert (kk == keys_before[k][inv]).all()
    obs, subj = v.tables()
    r0 = v.getRing(0)
    assert (obs[r0[:-1], 0] == r0[1:]).all() and obs[r0[-1], 0] == r0[0]
    assert (subj[r0[1:], 0] == r0[:-1]).all()
