"""FastPaxos fast-round tally on the GPU vs the reference's FastPaxosWithoutFallbackTests tables
(rapid/src/test/java/com/vrg/rapid/FastPaxosWithoutFallbackTests.java:85-90, :129-148), vs the oracle, and vs
plainref.FastRound on host-array streams that span many blocks of the tally kernel."""
import numpy as np
import pytest

import plainref

pytestmark = pytest.mark.gpu

NO_CONFLICTS = [(6, 5), (48, 37), (50, 38), (100, 76), (102, 77), (5, 4), (51, 39), (49, 37), (99, 75), (101, 76)]
CONFLICTS = [
    (6, 5, 1, True), (48, 37, 1, True), (50, 38, 1, True), (100, 76, 1, True), (102, 77, 1, True),
    (48, 37, 11, True), (50, 38, 12, True), (100, 76, 24, True), (102, 77, 25, True),
    (6, 5, 2, False), (48, 37, 14, False), (50, 38, 13, False), (100, 76, 25, False), (102, 77, 26, False),
]
CFG = 77


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.mark.parametrize("N,quorum", NO_CONFLICTS)
def test_fast_quorum_no_conflicts_vote_by_vote(rb, N, quorum):
    assert rb.quorum(N) == quorum
    fp = rb.FastPaxos(CFG, N, sender_capacity=N + 8)
    h1, h2 = rb.proposal_fingerprint([1235])
    for i in range(quorum - 1):
        r = fp.handleFastRoundProposals([i], [h1], [h2], [1])
        assert not r.decided and r.votes_received == i + 1
    r = fp.handleFastRoundProposals([quorum - 1], [h1], [h2], [1])
    assert r.decided and (r.hash, r.hash2, r.length) == (h1, h2, 1) and r.count == quorum and r.votes_received == quorum
    r = fp.handleFastRoundProposals([quorum], [h1], [h2], [1])           # after the decision: ignored (:138)
    assert r.decided and r.votes_received == quorum and r.count == quorum


@pytest.mark.parametrize("N,quorum,conflicts,change", CONFLICTS)
def test_fast_quorum_with_conflicts_one_call(rb, N, quorum, conflicts, change):
    """the whole vote sequence of the Java test as ONE array: decision point recovered by the prefix scan"""
    fp = rb.FastPaxos(CFG, N, sender_capacity=N + 8)
    p, c = rb.proposal_fingerprint([1235]), rb.proposal_fingerprint([1236])
    non_conflict = min(conflicts + quorum - 1, N - 1)
    senders = list(range(non_conflict + 1))
    h1 = [c[0]] * conflicts + [p[0]] * (non_conflict + 1 - conflicts)
    h2 = [c[1]] * conflicts + [p[1]] * (non_conflict + 1 - conflicts)
    r = fp.handleFastRoundProposals(senders, h1, h2, [1] * len(senders))
    assert r.decided == change
    if change:
        assert (r.hash, r.hash2) == p and r.count == quorum and r.votes_received == conflicts + quorum


def test_filters_dedupe_and_order(orc, rb):
    """random vote streams (duplicate senders, wrong configuration ids, several proposals, chunked calls) vs the oracle"""
    rng = np.random.default_rng(12)
    for trial in range(12):
        N = int(rng.integers(5, 120))
        cap = N + 20
        nprop = int(rng.integers(1, 4))
        props = [sorted(rng.choice(1000, size=int(rng.integers(1, 6)), replace=False).tolist()) for _ in range(nprop)]
        fps = [rb.proposal_fingerprint(p) for p in props]
        nv = int(rng.integers(1, 3 * N))
        senders = rng.integers(0, cap, size=nv).astype(np.int32)
        pid = rng.choice(nprop, size=nv, p=np.array([0.8] + [0.2 / max(1, nprop - 1)] * (nprop - 1)) if nprop > 1 else None)
        vcfg = np.where(rng.random(nv) < 0.1, CFG + 1, CFG).astype(np.int64)
        u = orc.Universe()
        stags = [u.add("s", int(s)) for s in range(cap)]
        ptags = {i: [u.add("p", int(x)) for x in props[i]] for i in range(nprop)}
        ofp = orc.FastPaxosTally(u, CFG, N)
        gfp = rb.FastPaxos(CFG, N, sender_capacity=cap)
        pos = 0
        while pos < nv:
            step = int(rng.integers(1, nv + 1))
            sl = slice(pos, min(nv, pos + step))
            for v in range(sl.start, sl.stop):
                ofp.handleFastRoundProposal(stags[senders[v]], int(vcfg[v]), ptags[int(pid[v])])
            r = gfp.handleFastRoundProposals(senders[sl], [fps[i][0] for i in pid[sl]], [fps[i][1] for i in pid[sl]],
                                             [len(props[i]) for i in pid[sl]], vote_cfg=vcfg[sl])
            assert r.decided == ofp.decided(), (trial, pos)
            assert r.votes_received == ofp.votesReceived(), (trial, pos)
            if r.decided:
                dec = [int(x) for x in ofp.decision()]
                want = [i for i in range(nprop) if ptags[i] == dec][0]
                assert (r.hash, r.hash2, r.length) == (fps[want][0], fps[want][1], len(props[want]))
                assert r.count == rb.quorum(N)
            pos = sl.stop


def test_bad_sender_rejected(rb):
    fp = rb.FastPaxos(CFG, 10, sender_capacity=10)
    with pytest.raises(rb.RapidError):
        fp.handleFastRoundProposals([10], [1], [1], [1])


def test_a_refused_call_leaves_no_trace(rb):
    """a call that is refused (a sender id outside the table) must not poison the tally: the senders it named can still vote;
    with 50,000 good votes the bad sender sits in a later block than the good ones"""
    for N, n_good in [(40, 10), (100_000, 50_000)]:
        fp = rb.FastPaxos(7, N, sender_capacity=N)
        good = np.arange(n_good, dtype=np.int32)
        with pytest.raises(rb.RapidError) as e:
            fp.handleFastRoundProposals(np.concatenate([good, [N + 5]]).astype(np.int32), np.full(n_good + 1, 99, np.uint64))
        assert e.value.code == rb._native.EINVAL and "vote %d:" % n_good in str(e.value), N
        q = rb.quorum(N)
        t = fp.handleFastRoundProposals(np.arange(q, dtype=np.int32), np.full(q, 99, np.uint64))
        assert t.decided and t.count == q and t.votes_received == q, N   # the good senders were NOT burnt by the refused call


def test_tally_from_cluster(orc, rb):
    """C2 end to end on one GPU: alert batch -> per-node proposals -> votes -> decision == the crashed set"""
    from helpers import OracleWorld
    from rapid_b200 import workloads as W
    n, K = 2000, 10
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    obs, _ = v.tables()
    b = W.c2_simultaneous_crash(obs, n, 0.01)
    for kernel in ("sweep", "bucketed"):
        cl = rb.VirtualCluster(v, 9, 4, kernel=kernel)
        blocked = W.blocked_by_receiver(b.blocked, v.getRing(0), 0, n)
        cfg = v.getCurrentConfigurationId(w.id_high, w.id_low)
        cl.handleBatch(cfg, b.src, b.dst, b.ring, b.status, blocked=blocked)
        fp = rb.FastPaxos(cfg, n)
        r = fp.tallyCluster(cl)
        want = rb.proposal_fingerprint(b.expected_cut)
        assert r.decided and (r.hash, r.hash2, r.length) == (want[0], want[1], 20)
        assert r.count == rb.quorum(n) and r.votes_received == rb.quorum(n)   # 1980 voters, decision at the 1501st


def test_empty_calls_and_reset(rb):
    fp = rb.FastPaxos(CFG, 9, sender_capacity=16)
    r = fp.handleFastRoundProposals([], [])
    assert not r.decided and r.votes_received == 0
    h = rb.proposal_fingerprint([3, 4])
    r = fp.handleFastRoundProposals(list(range(7)), [h[0]] * 7, [h[1]] * 7, [2] * 7)       # quorum of 9 is 7
    assert r.decided and r.count == 7
    fp.reset(CFG + 1)
    r = fp.handleFastRoundProposals(list(range(6)), [h[0]] * 6, [h[1]] * 6, [2] * 6, vote_cfg=[CFG + 1] * 6)
    assert not r.decided and r.votes_received == 6
    r = fp.handleFastRoundProposals([6], [h[0]], [h[1]], [2], vote_cfg=[CFG])                # stale configuration id
    assert not r.decided and r.votes_received == 6
    r = fp.handleFastRoundProposals([6], [h[0]], [h[1]], [2], vote_cfg=[CFG + 1])
    assert r.decided and r.votes_received == 7 and (r.hash, r.hash2, r.length) == (h[0], h[1], 2)
    r = fp.handleFastRoundProposals([99], [h[0]], [h[1]], [2], vote_cfg=[CFG + 1])                # after the decision: not checked
    assert r.decided and r.votes_received == 7 and r.count == 7 and (r.hash, r.hash2, r.length) == (h[0], h[1], 2)


def test_many_distinct_proposals_never_decide(rb):
    """every voter proposes something else (the conflict regime of the K,H,L sensitivity study): table growth, no decision"""
    n = 3000
    fp = rb.FastPaxos(CFG, n)
    hs = np.array([rb.proposal_fingerprint([i, i + 1]) for i in range(n)], dtype=np.uint64)
    r = fp.handleFastRoundProposals(np.arange(n), hs[:, 0], hs[:, 1], np.full(n, 2))
    assert not r.decided and r.votes_received == n


# ---------------------------------------------------------------- host-array streams over many blocks vs plainref.FastRound -------
BLOCK = 256                 # k_fp_tally gives every block a multiple of 256 votes
SPAN = 1536                 # ... and 1,536 of 10^6 votes on an H100 SXM (132 SMs x 5 co-resident blocks)


def _vote_stream(rb, rng, nv, cap, weights, p_stale=0.05):
    """nv votes by senders drawn with repeats from [0, cap), proposal k with weight weights[k], a fraction p_stale of them for
    the next configuration"""
    props = [tuple(rb.proposal_fingerprint(list(range(100 * k, 100 * k + k + 1)))) + (k + 1,) for k in range(len(weights))]
    pid = rng.choice(len(weights), size=nv, p=weights)
    table = np.array(props, np.uint64)
    return dict(senders=rng.integers(0, cap, size=nv).astype(np.int32), pid=pid, props=props, h1=table[pid, 0], h2=table[pid, 1],
                ln=table[pid, 2].astype(np.int32), vcfg=np.where(rng.random(nv) < p_stale, CFG + 1, CFG).astype(np.int64))


def _tally(fp, v, sl=slice(None)):
    return fp.handleFastRoundProposals(v["senders"][sl], v["h1"][sl], v["h2"][sl], v["ln"][sl], vote_cfg=v["vcfg"][sl])


def _ref_call(ref, v, sl=slice(None)):
    """the reference has no configuration ids: the stale votes are dropped before it sees them; returns the kept indices"""
    keep = np.nonzero(v["vcfg"][sl] == CFG)[0]
    ref.call(v["senders"][sl][keep], [v["props"][p] for p in v["pid"][sl][keep].tolist()])
    return keep


def _same(t, ref, what):
    assert t.decided == ref.decided, what
    assert t.votes_received == ref.votes_received, what
    if ref.decided:
        assert (t.hash, t.hash2, t.length) == ref.decision and t.count == ref.count, what


def _first_votes(v, sl=slice(None)):
    """index (within sl) of every sender's first vote of this configuration"""
    ok = np.nonzero(v["vcfg"][sl] == CFG)[0]
    s, first = np.unique(v["senders"][sl][ok], return_index=True)
    return s, ok[first]


@pytest.mark.parametrize("nv", [100_000, 1_000_000])
def test_multi_block_stream_one_call(rb, nv):
    """one call of nv votes by senders that vote again in later blocks, two proposals 80 : 20, stale votes mixed in: the quorum
    is reached mid-array inside a later block, and the first votes of new senders after it are not counted"""
    N = 2 * nv // 5
    cap = 2 * N
    v = _vote_stream(rb, np.random.default_rng(nv), nv, cap, [0.8, 0.2])
    ref = plainref.FastRound(N)
    keep = _ref_call(ref, v)
    assert ref.decided
    i_star = int(keep[ref.decided_at[1]])
    assert i_star >= 4 * SPAN and i_star % BLOCK not in (0, BLOCK - 1)          # inside a later block, not at its edge
    s, first = _first_votes(v)
    assert (first > i_star).sum() > 1000                                         # new senders after the decision
    ok = np.nonzero(v["vcfg"] == CFG)[0]
    late = ok - first[np.searchsorted(s, v["senders"][ok])] > 2 * SPAN
    assert (ok[late] < i_star).sum() > 1000                                       # repeats blocks after the first vote
    fp = rb.FastPaxos(CFG, N, sender_capacity=cap)
    t = _tally(fp, v)
    _same(t, ref, "decision")
    assert t.votes_received == (first <= i_star).sum() < len(s)
    _same(_tally(fp, v, slice(0, 1000)), ref, "after the decision")


def test_multi_block_stream_three_calls(rb):
    """the same stream in three calls: the first two stay below the quorum (repeats of their senders in later calls are
    ignored), the third reaches it mid-array inside a later block"""
    nv = 1_000_000
    N = 2 * nv // 5
    cap = 2 * N
    v = _vote_stream(rb, np.random.default_rng(3), nv, cap, [0.8, 0.2])
    cuts = [0, nv // 5 + 77, 2 * nv // 5 + 131, nv]
    fp = rb.FastPaxos(CFG, N, sender_capacity=cap)
    ref = plainref.FastRound(N)
    for c in range(3):
        sl = slice(cuts[c], cuts[c + 1])
        keep = _ref_call(ref, v, sl)
        assert ref.decided == (c == 2), c
        _same(_tally(fp, v, sl), ref, c)
    i_star = int(keep[ref.decided_at[1]])
    assert ref.decided_at[0] == 2 and i_star >= 4 * SPAN and i_star % BLOCK not in (0, BLOCK - 1)


def test_more_than_8_proposals_reaching_the_quorum_refuse_the_call(rb):
    """N = 5 (quorum 4): 9 proposals with 4 senders each cross the quorum in one call, which is refused and leaves no trace:
    the same senders then decide one proposal with exactly the quorum"""
    fp = rb.FastPaxos(CFG, 5, sender_capacity=40)
    hs = [rb.proposal_fingerprint([k]) for k in range(9)]
    senders = np.arange(36, dtype=np.int32)
    with pytest.raises(rb.RapidError) as e:
        fp.handleFastRoundProposals(senders, [hs[k // 4][0] for k in range(36)], [hs[k // 4][1] for k in range(36)], [1] * 36)
    assert e.value.code == rb._native.EUNSUPPORTED
    again = [35, 2, 17, 8, 30]                      # one sender from each of five groups; the fourth vote decides
    r = fp.handleFastRoundProposals(again, [hs[8][0]] * 5, [hs[8][1]] * 5, [1] * 5)
    assert r.decided and (r.hash, r.hash2, r.length) == (hs[8][0], hs[8][1], 1)
    assert r.count == 4 and r.votes_received == 4
