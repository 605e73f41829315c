"""The classic-Paxos fallback (csrc/classic_paxos.cu) at the sizes where the device code takes paths the small cases never
reach, field by field against tests/plainref.py (pinned against the oracle's literal instances on CPU by
tests/test_oracle_classic_paxos_vs_plainref.py):

* the coordinator rule from 1 to 10^6 messages: one and several 4,096-pair sort tiles, the 16 -> 17-bit key width at
  16,384 -> 16,385 messages, 1 to ~m/3 distinct values, (N/4 + 1)-th occurrences of two values at adjacent arrivals on both
  sides of a tile edge, values that collide in the warp fold at adjacent lanes;
* the Phase1b list growing far past message_capacity across calls, the trigger in a later call, a second startPhase1a;
* the Phase2b table across calls with many rounds and repeated senders, and the refusal at pairs + 2n > 3T/4;
* 10^6 acceptors with Zipf-spread fast-round votes, competing coordinators, both arrival orders, a learner;
* registration of the detector's votes at 10^5 receivers, and an acceptor listed twice in one registration."""
import numpy as np
import pytest

import plainref as P
from test_oracle_classic_paxos_vs_plainref import rule_list, value_pool

pytestmark = pytest.mark.gpu

CFG = 1


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


def triple(h1, h2, ln, i):
    return (int(h1[i]), int(h2[i]), int(ln[i]))


# ------------------------------------------------------------------------------------------------ the stateless rule
SIZES = [1, 4095, 4096, 4097, 16384, 16385, 100_000, 1_000_000]
RULE_CASES = sorted({(m, min(v, m)) for m in SIZES for v in (1, 2, 300, 5000, max(1, m // 3))})


@pytest.mark.parametrize("m,n_values", RULE_CASES)
def test_rule_matches_plainref(rb, m, n_values):
    rng = np.random.default_rng(m * 7 + n_values)
    vr, h1, h2, ln, N = rule_list(rng, m, n_values)
    col = (P.pack_rank(vr) == P.pack_rank(vr).max()) & (ln > 0)
    cmax = int(np.bincount(P._value_ids(h1[col], h2[col], ln[col])).max()) if col.any() else 1
    # the drawn N, and one whose N/4 + 1 is reached by the most frequent collected value
    for n in (N, 4 * max(0, int(cmax * 0.7)) + 2):
        px = rb.Paxos(CFG, n, message_capacity=64)
        want = P.coordinator_rule(n, vr, h1, h2, ln)
        assert px.selectProposalUsingCoordinatorRule(vr, h1, ln, h2) == want, (n, want)
        px.close()


def adjacent_kth(rng, m, edge, a_first):
    """values A and B reach their N/4 + 1-th occurrence at arrivals edge - 1 and edge (A first or B first); the arrivals
    before hold N/4 copies of each, many other values (fewer copies each), empty vvals and lower ranks"""
    need = 700
    nv = max(400, edge // 50)
    ph1, ph2, pln = value_pool(nv, 3)
    vi = 8 + rng.integers(0, nv - 8, size=m)
    lo = np.arange(edge - 1)
    ab = rng.permutation(lo)[: 2 * (need - 1)]
    vi[ab[: need - 1]], vi[ab[need - 1:]] = 0, 4
    vi[edge - 1], vi[edge] = (0, 4) if a_first else (4, 0)
    tail = np.arange(edge + 1, m)
    vi[tail[rng.random(len(tail)) < 0.3]] = 0
    h1, h2, ln = ph1[vi], ph2[vi], pln[vi].copy()
    vr = np.tile(np.array([[2, 7]], np.int64), (m, 1))
    other = np.nonzero((vi >= 8) & (rng.random(m) < 0.2))[0]
    vr[other[: len(other) // 2]] = (2, 6)
    ln[other[len(other) // 2:]] = 0
    return vr, h1, h2, ln, 4 * (need - 1) + 1


@pytest.mark.parametrize("m,edge", [(4097, 4096), (16385, 4096), (16385, 8192), (1_000_000, 4096), (1_000_000, 1 << 19)])
@pytest.mark.parametrize("a_first", [True, False])
def test_rule_adjacent_kth_across_tile_edge(rb, m, edge, a_first):
    rng = np.random.default_rng(edge + m + a_first)
    vr, h1, h2, ln, N = adjacent_kth(rng, m, edge, a_first)
    assert P.coordinator_rule(N, vr, h1, h2, ln) == edge - 1
    px = rb.Paxos(CFG, N, message_capacity=64)
    assert px.selectProposalUsingCoordinatorRule(vr, h1, ln, h2) == edge - 1


@pytest.mark.parametrize("m", [64, 4097, 100_000])
@pytest.mark.parametrize("swap", [False, True])
def test_rule_fold_collisions_in_one_warp(rb, m, swap):
    """two values with the same warp fold alternate at adjacent lanes: they are two values (not one), and the one whose
    N/4 + 1-th occurrence comes first wins"""
    ph1, ph2, pln = value_pool(4, 11)
    x, y = (3, 0) if swap else (0, 3)
    vi = np.where(np.arange(m) % 2 == 0, x, y)
    h1, h2, ln = ph1[vi], ph2[vi], pln[vi]
    vr = np.tile(np.array([[1, 1]], np.int64), (m, 1))
    for need in (1, 2, 17, m // 4):
        N = 4 * (need - 1) + 3
        want = P.coordinator_rule(N, vr, h1, h2, ln)
        assert want == 2 * (need - 1)
        px = rb.Paxos(CFG, N, message_capacity=64)
        assert px.selectProposalUsingCoordinatorRule(vr, h1, ln, h2) == want


# ------------------------------------------------------------------------------------------------ Phase1b across calls
def phase1b_batch(rng, n, crnd, top_share, nonempty):
    ph1, ph2, pln = value_pool(2000, 21)
    zipf = 1.0 / np.arange(1, 2000) ** 1.2
    vi = np.where(rng.random(n) < top_share, 0, 1 + rng.choice(1999, size=n, p=zipf / zipf.sum()))
    h1, h2, ln = ph1[vi], ph2[vi], np.where(rng.random(n) < nonempty, pln[vi], 0)
    vr = np.where(rng.random(n)[:, None] < 0.8, np.array([1, 1]), np.array([0, 0])).astype(np.int64)
    rnd = np.tile(np.array(crnd, np.int64), (n, 1))
    stale = rng.random(n) < 0.05
    rnd[stale] = (1, 3)                                                # another coordinator's round
    cfg = np.where(rng.random(n) < 0.03, CFG + 1, CFG)                 # a stale configuration
    return rnd, vr, h1, h2, ln, cfg


@pytest.mark.parametrize("case", ["kth", "fallback", "late"])
def test_phase1b_list_grows_across_calls(rb, case):
    """N = 10^6, message_capacity = 1,000: batches of 3,000 to 300,000; the trigger (N/2 + 1 kept answers) falls in a later
    batch.  kth: the rule picks the value reaching N/4 + 1 occurrences; fallback: none does; late: every vval is empty until
    after N/2.  A second startPhase1a mid-stream moves crnd while the list persists."""
    N = 1_000_000
    rng = np.random.default_rng({"kth": 1, "fallback": 2, "late": 3}[case])
    px = rb.Paxos(CFG, N, message_capacity=1000)
    ref = P.Coordinator(N, CFG)
    assert px.startPhase1a(2, 5) and ref.startPhase1a(2, 5)
    crnd = (2, 5)
    sizes = [3000, 30_000, 300_000, 120_000, 3000, 300_000, 200_000]
    top = {"kth": 0.85, "fallback": 0.3, "late": 0.85}[case]
    proposed = 0
    for b, n in enumerate(sizes):
        if b == 3:
            assert px.startPhase1a(2, 8) and ref.startPhase1a(2, 8)
            crnd = (2, 8)
        nonempty = 0.0 if case == "late" and b < 6 else 0.85
        rnd, vr, h1, h2, ln, cfg = phase1b_batch(rng, n, crnd, top, nonempty)
        got = px.handlePhase1bMessages(rnd, vr, h1, ln, h2, msg_cfg=cfg)
        want = ref.handle(rnd, vr, h1, ln, h2, msg_cfg=cfg)
        assert (got.proposed, got.trigger_index, got.cval, got.n_messages) == want, (b, got, want)
        proposed += got.proposed
    assert proposed == 1 and ref.n_messages > N // 2


# ------------------------------------------------------------------------------------------------ Phase2b across calls
def phase2b_batch(rng, n, N, rounds, hot, senders):
    ph1, ph2, pln = value_pool(16, 31)
    ri = np.where(rng.random(n) < 0.5, hot, rng.integers(0, len(rounds), size=n))
    rk = np.array(rounds, np.int64)[ri]
    s = rng.integers(senders[0], senders[1], size=n)
    vi = rng.integers(0, 16, size=n)
    cfg = np.where(rng.random(n) < 0.02, CFG - 1, CFG)
    return rk, s, ph1[vi], ph2[vi], pln[vi], cfg


def test_phase2b_many_rounds_across_calls(rb):
    """10^6 messages in calls of 10^5 over 40 rounds, senders repeated within and across calls; the decision (N/2 + 1
    distinct senders in one round) comes in a later call, at the arrival plainref names, with that message's value"""
    N = 200_000
    rng = np.random.default_rng(5)
    rounds = [(2, int(x)) for x in rng.choice(np.arange(-1000, 1000), size=40, replace=False)]
    px = rb.Paxos(CFG, N, message_capacity=1_000_000)
    ref = P.Learner(N, CFG)
    decided_in = None
    for c in range(10):
        rk, s, h1, h2, ln, cfg = phase2b_batch(rng, 100_000, N, rounds, 7, (0, N + 1000))
        got = px.handlePhase2bMessages(rk, s, h1, ln, h2, msg_cfg=cfg)
        want = ref.handle(rk, s, h1, ln, h2, msg_cfg=cfg)
        assert (got.decided, got.decided_index, got.decision) == want, (c, got, want)
        if got.decided_index >= 0:
            decided_in = c
    assert decided_in is not None and decided_in >= 2


def test_phase2b_capacity_boundary(rb):
    """message_capacity 2^16 -> a table of 2^18 entries, refused past 3/4 of it: the largest call that fits is taken, one
    message more is refused with ENOMEM and changes nothing, and a following call that fits decides as plainref says"""
    N, cap = 60_000, 1 << 16
    limit = (1 << 18) // 4 * 3
    rng = np.random.default_rng(9)
    rounds = [(2, i) for i in range(12)]
    px = rb.Paxos(CFG, N, message_capacity=cap)
    ref = P.Learner(N, CFG)

    def call(rk, s, h1, h2, ln, cfg):
        got = px.handlePhase2bMessages(rk, s, h1, ln, h2, msg_cfg=cfg)
        want = ref.handle(rk, s, h1, ln, h2, msg_cfg=cfg)
        assert (got.decided, got.decided_index, got.decision) == want
        return got

    def refused(n, senders):
        with pytest.raises(rb.RapidError) as e:
            rk, s, h1, h2, ln, cfg = phase2b_batch(rng, n, N, rounds, 0, senders)
            px.handlePhase2bMessages(rk, s, h1, ln, h2, msg_cfg=cfg)
        assert e.value.code == rb._native.ENOMEM

    call(*phase2b_batch(rng, 40_000, N, rounds, 0, (0, 29_000)))       # half of it in round 0, from 29,000 senders
    assert not ref.decided
    fit = (limit - ref.entries) // 2
    refused(fit + 1, (0, 29_000))
    call(*phase2b_batch(rng, fit, N, rounds, 0, (0, 29_000)))          # exactly the largest call that fits
    assert not ref.decided
    fit = (limit - ref.entries) // 2
    assert fit > 0
    refused(fit + 1, (0, N))
    got = call(*phase2b_batch(rng, fit, N, rounds, 0, (0, N)))
    assert got.decided and got.decided_index >= 0


# ------------------------------------------------------------------------------------------------ from acceptors at 10^6
def zipf_votes(n, seed):
    """about 80 % of n acceptors vote, over 3,000 values with a Zipf-like spread (the most popular value just clears N/4 + 1
    among the first N/2 + 1 answers); acceptors 0-49 do not vote and acceptor 50 votes for a value other than the most
    popular one -> (acceptors, h1, h2, len)"""
    rng = np.random.default_rng(seed)
    ph1, ph2, pln = value_pool(3000, seed)
    zipf = 1.0 / np.arange(1, 3000) ** 1.3
    vi = np.where(rng.random(n) < 0.64, 0, 1 + rng.choice(2999, size=n, p=zipf / zipf.sum()))
    vi[50] = 5
    voters = np.nonzero((rng.random(n) < 0.8) & (np.arange(n) >= 50) | (np.arange(n) == 50))[0]
    return voters, ph1[vi[voters]], ph2[vi[voters]], pln[vi[voters]]


def same1(got, want):
    assert (got.proposed, got.trigger_index, got.cval, got.n_messages) == want, (got, want)


def same2(got, want):
    assert (got.decided, got.decided_index, got.decision) == want, (got, want)


def same_registers(acc, ref, rng, extra=()):
    R = ref.R
    for r in sorted(set(rng.choice(R, size=min(R, 1000), replace=False).tolist()) | {0, R - 1} | set(extra)):
        assert acc.read(r) == ref.read(r), r


def test_one_million_acceptors_against_plainref(rb):
    """Zipf-spread votes on 10^6 acceptors; coordinator a at (2, 5) takes its answers in acceptor order, coordinator b at
    (2, 9) pre-empts it and takes its answers in a permuted order (and c at (2, 9) the same answers in acceptor order); a's
    Phase2a is then rejected everywhere, b's accepted everywhere; learners in both orders"""
    n = 1_000_000
    rng = np.random.default_rng(17)
    acc, ref = rb.PaxosAcceptors(CFG, n), P.Acceptors(CFG, n)
    voters, h1, h2, ln = zipf_votes(n, 3)
    acc.registerFastRoundVotes(voters, h1, ln, h2)
    ref.registerFastRoundVotes(voters, h1, ln, h2)
    same_registers(acc, ref, rng)
    coords = {k: (rb.Paxos(CFG, n, message_capacity=n), P.Coordinator(n, CFG)) for k in "abc"}
    for k, node in (("a", 5), ("b", 9), ("c", 9)):
        assert coords[k][0].startPhase1a(2, node) and coords[k][1].startPhase1a(2, node)
    assert acc.handlePhase1aMessage((2, 5)) == ref.phase1a((2, 5)) == n
    same1(coords["a"][0].handlePhase1bFromAcceptors(acc, 0), ref.deliver1b(coords["a"][1], 0))
    assert acc.handlePhase1aMessage((2, 9)) == ref.phase1a((2, 9)) == n
    seed = 0x5EED_0F_0B
    for k, perm in (("b", seed), ("c", 0), ("a", seed)):               # a: answers to another rank, all dropped
        same1(coords[k][0].handlePhase1bFromAcceptors(acc, perm), ref.deliver1b(coords[k][1], perm))
    assert coords["b"][1].cval is not None and coords["a"][1].n_messages == n
    assert acc.handlePhase2aMessage((2, 5), coords["a"][1].cval) == ref.phase2a((2, 5), coords["a"][1].cval) == 0
    assert acc.handlePhase2aMessage((2, 9), coords["b"][1].cval) == ref.phase2a((2, 9), coords["b"][1].cval) == n
    same_registers(acc, ref, rng)
    for perm in (0, 4242):
        same2(rb.Paxos(CFG, n, message_capacity=n).handlePhase2bFromAcceptors(acc, perm), ref.deliver2b(P.Learner(n, CFG), perm))


# ------------------------------------------------------------------------------------------------ registration
def test_register_votes_from_cluster_at_1e5(rb):
    """10^5 receivers, bitmap delivery: groups of receivers miss one crashed subject's alerts, or half of one, so the
    detector yields several distinct proposals and some receivers announce nothing; a host-list vote registered before
    stays only where the receiver did not announce"""
    from rapid_b200 import workloads as W
    n, K, H, L = 100_000, 10, 9, 4
    view = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    obs, _ = view.tables()
    subjects = [11, 20_202, 50_005, 99_000]
    cells = [(int(obs[s][k]), s, k) for s in subjects for k in range(K)]
    src, dst, ring = (np.array(x) for x in zip(*cells))
    group = np.arange(n) % 6                                           # group g < 4 misses subject g; 5 misses half of 0
    mask = np.ones((len(cells), n), bool)
    for c, (_, s, k) in enumerate(cells):
        g = subjects.index(s)
        mask[c, group == g] = False
        if g == 0 and k < 5:
            mask[c, group == 5] = False
    words = (n + 31) // 32
    bits = np.zeros((len(cells), words * 32), bool)
    bits[:, :n] = mask
    bm = np.packbits(bits, axis=1, bitorder="little").view("<u4")
    cfg = view.getCurrentConfigurationId(*W.node_ids(0, n))
    cl = rb.VirtualCluster(view, H, L, kernel="bucketed")
    cl.handleBatch(cfg, src, dst, ring, np.ones(len(cells), np.uint8), bitmap=bm)
    out = cl.readOutputs()
    ann = np.asarray(out.announced).astype(bool)
    assert not ann[group == 5].any() and ann[group != 5].all()
    props = {(int(a), int(b), int(c)) for a, b, c in zip(out.proposal_hash[ann], out.proposal_hash2[ann], out.proposal_len[ann])}
    assert len(props) == 5
    acc, ref = rb.PaxosAcceptors(cfg, n), P.Acceptors(cfg, n)
    pre = np.arange(0, n, 7)
    ph1, ph2, pln = value_pool(4, 77)
    acc.registerFastRoundVotes(pre, ph1[pre % 4], pln[pre % 4], ph2[pre % 4])
    ref.registerFastRoundVotes(pre, ph1[pre % 4], pln[pre % 4], ph2[pre % 4])
    acc.registerFastRoundVotesFrom(cl)
    ref.registerFrom(out.proposal_hash, out.proposal_hash2, out.proposal_len, ann)
    rng = np.random.default_rng(4)
    same_registers(acc, ref, rng, extra=[5, 35, 11, 17, 23, 29])       # group 5, pre-registered or not


def test_acceptor_listed_twice_keeps_its_last_vote(rb):
    """one registration call names acceptor 40 at adjacent entries and acceptor 7 about 10^6 entries apart, each time with
    another vote: both end with their last listed vote, all five fields, as one-by-one calls in list order would leave them"""
    R = 1_000_100
    rng = np.random.default_rng(12)
    order = rng.permutation(R)
    order = order[(order != 7) & (order != 40)]
    lst = np.concatenate([[7], order[:500], [40, 40], order[500:], [7]]).astype(np.int64)
    n = len(lst)
    ph1, ph2, pln = value_pool(8, 99)
    vi = rng.integers(0, 8, size=n)
    first40 = 1 + 500
    vi[0], vi[n - 1] = 1, 2                                            # acceptor 7: values differing only in hash2
    vi[first40], vi[first40 + 1] = 4, 6                                # acceptor 40: values differing only in len
    assert first40 // 32 == (first40 + 1) // 32                        # the two entries share a warp
    acc, ref = rb.PaxosAcceptors(CFG, R), P.Acceptors(CFG, R)
    acc.registerFastRoundVotes(lst, ph1[vi], pln[vi], ph2[vi])
    ref.registerFastRoundVotes(lst, ph1[vi], pln[vi], ph2[vi])
    assert acc.read(7) == {"rnd": (1, 1), "vrnd": (1, 1), "vval": triple(ph1, ph2, pln, 2)}
    assert acc.read(40) == {"rnd": (1, 1), "vrnd": (1, 1), "vval": triple(ph1, ph2, pln, 6)}
    same_registers(acc, ref, rng, extra=[7, 40] + order[:20].tolist())
    # a list naming an acceptor out of range is refused and changes no acceptor
    with pytest.raises(rb.RapidError) as e:
        acc.registerFastRoundVotes([7, 40, R], ph1[:3], pln[:3], ph2[:3])
    assert e.value.code == rb._native.EINVAL
    same_registers(acc, ref, rng, extra=[7, 40])
