"""The device view change (csrc/view.cu: apply_cut_device, DESIGN §4.8) against two references at sizes the oracle cannot reach:
plainref.view_change (NumPy, from the keys before the cut) and a view built afresh from the post-cut endpoint list (build_rings).
Every ring, every key, the observer / subject tables and the configuration id are compared in full.

The joiners of a cut are ranked by an all-pairs kernel up to 32,768 of them and by per-ring radix sorts above that; the cases
cover both sides of that edge, duplicate endpoints among the joiners on both sides, and refused cuts, which must leave the view
bit-identical, identifiersSeen included.  The CPU test pins plainref.view_change against the oracle's ringDelete / ringAdd."""
import numpy as np
import pytest

import plainref
from helpers import OracleWorld
from rapid_b200 import workloads as W

K = 10
RANK_LIMIT = 32768          # apply_cut_device: all-pairs rank up to here, per-ring radix sorts above


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


# ---------------------------------------------------------------- the reference itself, against the oracle (CPU) ------------------
# seeds 0-15 draw K from {3, 7, 10}; seeds 16-17 fix it at the largest ring count
@pytest.mark.parametrize("seed,K14", [(s, False) for s in range(16)] + [(16, True), (17, True)],
                         ids=[str(s) for s in range(16)] + ["16-K14", "17-K14"])
def test_plain_view_change_matches_oracle(orc, seed, K14):
    rng = np.random.default_rng(900 + seed)
    Kx = int(rng.choice([3, 7, 10]))
    if K14:
        Kx = 14
    n = int(rng.integers(0, 60))
    nj = int(rng.integers(0, 20))
    w = OracleWorld(orc, n, Kx, n_joiners=nj)
    tot = n + nj
    keys = np.array([[w.view.key(k, t) for t in range(tot)] for k in range(Kx)], np.int64).reshape(Kx, tot)
    leave = rng.choice(n, size=int(rng.integers(0, n + 1)), replace=False) if n else np.zeros(0, np.int64)
    join = n + rng.choice(nj, size=int(rng.integers(0, nj + 1)), replace=False) if nj else np.zeros(0, np.int64)
    cut = rng.permutation(np.concatenate([leave, join]).astype(np.int64))
    ref = plainref.view_change(keys, n, cut)
    hi, lo = W.node_ids(n, nj)
    for x in sorted(leave.tolist()):
        w.view.ringDelete(x)
    for x in sorted(join.tolist()):
        w.view.ringAdd(x, (int(hi[x - n]), int(lo[x - n])))
    kept = ref.kept
    assert w.view.getMembershipSize() == len(kept)
    assert sorted(kept.tolist()) == sorted(set(range(n)) - set(leave.tolist()) | set(join.tolist()))
    assert (ref.old_to_new[kept] == np.arange(len(kept))).all() and (np.diff(kept) > 0).all()
    for k in range(Kx):
        assert kept[ref.rings[k]].tolist() == w.view.getRing(k)
    # tables from a view built afresh on the new membership (the oracle's changed view answers from a cache, DESIGN §7)
    fresh = orc.MembershipView(w.u, Kx, kept.astype(np.int32), hi[:0], lo[:0])
    if len(kept) > 1:
        o_obs, o_subj = fresh.tables(kept.astype(np.int32))
        np.testing.assert_array_equal(kept[ref.obs], o_obs)
        np.testing.assert_array_equal(kept[ref.subj], o_subj)
    with pytest.raises(ValueError):
        plainref.view_change(keys, n, [0, 0] if tot else [0])


def test_plain_view_change_reports_equal_keys():
    keys = np.array([[5, -3, 9, 9], [1, 2, 3, 4]], np.int64)
    with pytest.raises(plainref.RingCollision) as e:
        plainref.view_change(keys, 2, [2, 3])
    assert (e.value.ring, {e.value.a, e.value.b}) == (0, {2, 3})
    assert plainref.view_change(keys, 2, [3]).rings[0].tolist() == [1, 0, 2]


# ---------------------------------------------------------------- the device view change ------------------------------------------
class Tracked:
    """A device view plus what the tests know about it: the endpoint (index into a pool of synthetic endpoints) and NodeId of
    every id, and identifiersSeen."""

    def __init__(self, rb, n, pool, K=K):
        self.rb, self.K = rb, K
        self.hb, self.off, self.ports = W.packed_endpoints(0, pool)
        self.pool_hi, self.pool_lo = W.node_ids(0, pool)
        self.v = rb.MembershipView.from_packed(self.K, *self.packed(np.arange(n)))
        self.ep = np.arange(n)
        self.hi, self.lo = self.pool_hi[:n].copy(), self.pool_lo[:n].copy()
        self.v.setNodeIds(self.hi, self.lo)
        self.seen_hi, self.seen_lo = self.hi.copy(), self.lo.copy()
        self.next = n                                   # first pool endpoint never used

    def packed(self, ep):
        ep = np.asarray(ep, np.int64)
        lens = (self.off[ep + 1] - self.off[ep]).astype(np.int64)
        off = np.zeros(len(ep) + 1, np.int32)
        np.cumsum(lens, out=off[1:])
        src = np.repeat(self.off[ep].astype(np.int64) - off[:-1], lens) + np.arange(int(off[-1]))
        hb = self.hb[src] if len(src) else np.zeros(1, np.uint8)
        return hb, off, self.ports[ep]

    def fresh_endpoints(self, count):
        ep = np.arange(self.next, self.next + count)
        self.next += count
        return ep

    def register(self, ep, hi=None, lo=None):
        """register pool endpoints `ep` as joiners, NodeIds hi/lo (default: the endpoints' own)"""
        ep = np.asarray(ep, np.int64)
        hi = self.pool_hi[ep] if hi is None else np.asarray(hi, np.int64)
        lo = self.pool_lo[ep] if lo is None else np.asarray(lo, np.int64)
        hosts = [bytes(self.hb[self.off[e]: self.off[e + 1]]) for e in ep.tolist()]
        first = self.v.registerJoiners(hosts, self.ports[ep])[0]
        assert first == len(self.ep)
        self.v.setJoinerIds(first, hi, lo)
        self.ep = np.concatenate([self.ep, ep])
        self.hi, self.lo = np.concatenate([self.hi, hi]), np.concatenate([self.lo, lo])
        return np.arange(first, first + len(ep))

    def state(self):
        """everything a refused cut must leave as it was"""
        v = self.v
        obs, subj = v.tables()
        return (v.getMembershipSize(), v.numJoiners(), [v.getRing(k).tolist() for k in range(self.K)],
                [v.keys(k).tolist() for k in range(self.K)], obs.tolist(), subj.tolist(), v.joinerTables().tolist(),
                v.currentConfigurationId())

    def refused(self, cut, exc):
        before = self.state()
        with pytest.raises(exc):
            self.v.applyCut(cut)
        assert self.state() == before

    def apply(self, cut):
        """apply `cut` on the device and compare the result with both references"""
        v, K = self.v, self.K
        n = v.getMembershipSize()
        assert n + v.numJoiners() == len(self.ep)
        keys = np.stack([v.keys(k) for k in range(K)]) if len(self.ep) else np.zeros((K, 0), np.int64)
        ref = plainref.view_change(keys, n, cut)
        mapping = v.applyCut(np.asarray(cut, np.int32))
        np.testing.assert_array_equal(mapping, ref.old_to_new)
        n2 = len(ref.kept)
        assert v.getMembershipSize() == n2 and v.numJoiners() == 0
        for k in range(K):
            np.testing.assert_array_equal(v.getRing(k), ref.rings[k], err_msg="ring %d" % k)
            np.testing.assert_array_equal(v.keys(k), ref.keys[k], err_msg="keys of ring %d" % k)
        obs, subj = v.tables()
        np.testing.assert_array_equal(obs, ref.obs)
        np.testing.assert_array_equal(subj, ref.subj)
        admitted = ref.kept[ref.kept >= n]
        self.seen_hi = np.concatenate([self.seen_hi, self.hi[admitted]])
        self.seen_lo = np.concatenate([self.seen_lo, self.lo[admitted]])
        self.ep, self.hi, self.lo = self.ep[ref.kept], self.hi[ref.kept], self.lo[ref.kept]
        # the second reference: the same membership built from scratch (build_rings)
        fresh = self.rb.MembershipView.from_packed(K, *self.packed(self.ep))
        for k in range(K):
            np.testing.assert_array_equal(fresh.getRing(k), ref.rings[k], err_msg="fresh ring %d" % k)
            np.testing.assert_array_equal(fresh.keys(k), ref.keys[k])
        f_obs, f_subj = fresh.tables()
        np.testing.assert_array_equal(f_obs, obs)
        np.testing.assert_array_equal(f_subj, subj)
        assert v.currentConfigurationId() == fresh.getCurrentConfigurationId(self.seen_hi, self.seen_lo)
        return ref


@pytest.mark.gpu
@pytest.mark.parametrize("members", [1000, 200_000])
@pytest.mark.parametrize("m", [0, 1, RANK_LIMIT - 1, RANK_LIMIT, RANK_LIMIT + 1, 40_000])
def test_cut_admits_m_joiners(rb, members, m):
    """m joiners admitted (three more registered and left out) while 1 % of the members leave"""
    rng = np.random.default_rng(members + m)
    t = Tracked(rb, members, members + m + 3)
    jids = t.register(t.fresh_endpoints(m + 3))
    join = np.sort(rng.choice(jids, size=m, replace=False))
    leave = rng.choice(members, size=members // 100, replace=False)
    ref = t.apply(rng.permutation(np.concatenate([leave, join])))
    assert int((ref.kept >= members).sum()) == m            # m > RANK_LIMIT: the joiners were ranked by the radix sorts
    assert len(ref.kept) == members - members // 100 + m


@pytest.mark.gpu
@pytest.mark.parametrize("m", [100, RANK_LIMIT + 1])
def test_cut_at_fourteen_rings(rb, m):
    """the same cut at K = 14 on both sides of the rank / radix edge: 1 % of 5,000 members leave, m joiners come in"""
    rng = np.random.default_rng(14 + m)
    t = Tracked(rb, 5000, 5000 + m + 3, K=14)
    jids = t.register(t.fresh_endpoints(m + 3))
    join = np.sort(rng.choice(jids, size=m, replace=False))
    ref = t.apply(rng.permutation(np.concatenate([rng.choice(5000, size=50, replace=False), join])))
    assert int((ref.kept >= 5000).sum()) == m and len(ref.kept) == 5000 - 50 + m


@pytest.mark.gpu
def test_leaves_only_and_joins_only(rb):
    rng = np.random.default_rng(3)
    t = Tracked(rb, 5000, 5000 + 700)
    jids = t.register(t.fresh_endpoints(300))
    t.apply(rng.choice(5000, size=123, replace=False))               # leaves only: every registered joiner is dropped
    assert t.v.getMembershipSize() == 5000 - 123
    jids = t.register(t.fresh_endpoints(400))
    t.apply(jids[rng.permutation(len(jids))])                          # joins only
    assert t.v.getMembershipSize() == 5000 - 123 + 400
    t.apply([])                                                        # nothing at all
    del jids


@pytest.mark.gpu
@pytest.mark.parametrize("members,m", [(1, 1), (300, 40), (2000, 5000)])
def test_every_member_leaves_while_joiners_come_in(rb, members, m):
    t = Tracked(rb, members, members + m + 10)
    jids = t.register(t.fresh_endpoints(m + 10))
    ref = t.apply(np.concatenate([np.arange(members), jids[5: 5 + m]]))
    assert (ref.kept >= members).all() and len(ref.kept) == m          # no member survives (n_surv = 0)


@pytest.mark.gpu
def test_consecutive_cuts_cross_powers_of_two(rb):
    """one view, six cuts: its size crosses 1024, 2048, 4096 and 8192 up and down, so the key stride changes and the cut's
    scratch buffers are reused at other sizes"""
    rng = np.random.default_rng(11)
    t = Tracked(rb, 1000, 40_000)
    for add, drop in [(100, 0), (0, 200), (3000, 0), (300, 50), (0, 4000), (6000, 100)]:
        n = t.v.getMembershipSize()
        jids = t.register(t.fresh_endpoints(add + 7))
        join = rng.choice(jids, size=add, replace=False)
        t.apply(rng.permutation(np.concatenate([rng.choice(n, size=drop, replace=False), join])))
        assert t.v.getMembershipSize() == n - drop + add


@pytest.mark.gpu
def test_refused_cuts_leave_the_view_unchanged(rb):
    t = Tracked(rb, 600, 800)
    jids = t.register(t.fresh_endpoints(20))
    t.refused([5, 600 + 20], rb.RapidError)                                  # an id past the joiners
    t.refused([-1], rb.RapidError)
    t.refused([7, 9, 7], rb.NodeNotInRingException)                          # a member named twice: second ringDelete
    t.refused([int(jids[3]), 2, int(jids[3])], rb.NodeAlreadyInRingException)   # a joiner named twice: second ringAdd
    # a joiner whose NodeId is a member's: UUIDAlreadySeenException
    bad = t.register(t.fresh_endpoints(1), hi=[t.hi[17]], lo=[t.lo[17]])
    t.refused([1, int(jids[0]), int(bad[0])], rb.UUIDAlreadySeenException)
    # the same view still takes a good cut afterwards
    t.apply([1, 2, int(jids[0]), int(jids[5])])


def _duplicate_joiners(rb, m):
    """a 1000-member view with m registered joiners, the last of which repeats the endpoint of one in the middle; every joiner
    has its own NodeId, so the copies differ there.  -> (view, joiner ids, the two copies, a cut that admits both)"""
    rng = np.random.default_rng(m)
    t = Tracked(rb, 1000, 1000 + m)
    ep = t.fresh_endpoints(m - 1)
    ep = np.concatenate([ep, ep[m // 3: m // 3 + 1]])
    hi, lo = W.node_ids(10 ** 7, m)                                           # NodeIds nobody else has
    jids = t.register(ep, hi, lo)
    leave = rng.choice(1000, size=10, replace=False)
    return t, jids, (int(jids[m // 3]), int(jids[-1])), rng.permutation(np.concatenate([leave, jids]))


@pytest.mark.gpu
@pytest.mark.parametrize("m", [200, 40_000])
def test_duplicate_endpoint_among_the_joiners(rb, m):
    """a cut that admits the same endpoint twice is refused as the reference's second ringAdd would be
    (NodeAlreadyInRingException), on both sides of the rank / radix edge, and leaves the view as it was; a cut that admits one
    copy then succeeds"""
    t, jids, (a, b), cut = _duplicate_joiners(rb, m)
    assert len(jids) == m and (m > RANK_LIMIT) == (m == 40_000)
    t.refused(cut, rb.NodeAlreadyInRingException)
    ref = t.apply(cut[cut != a])
    assert ref.old_to_new[a] == -1 and ref.old_to_new[b] >= 0


@pytest.mark.gpu
def test_a_cut_refused_after_the_uuid_check_leaves_identifiers_seen_alone(rb):
    """the joiners' NodeIds pass the UUID rule before the rings are merged; when the merge then refuses the cut, identifiersSeen
    (and so the configuration id) must not have taken them, and a later cut may still admit those joiners"""
    t, jids, (a, b), cut = _duplicate_joiners(rb, 200)
    before = t.v.currentConfigurationId()
    with pytest.raises(rb.RapidError):
        t.v.applyCut(cut)
    assert t.v.currentConfigurationId() == before
    ref = t.apply(cut[cut != b])                                                 # UUIDAlreadySeenException if the ids stuck
    assert ref.old_to_new[b] == -1 and ref.old_to_new[a] >= 0
