"""GPU parity of the sharded classic-Paxos tallies (rapid_px_phase1b_from_acceptor_shards / _phase2b_, csrc/classic_paxos.cu):
the answers of several PaxosAcceptors shards, delivered to one coordinator / learner, must give bit for bit what the
single-handle call gives on one PaxosAcceptors holding the union of their acceptors — outputs and the state the Paxos keeps
for later calls alike.  Every case runs comm-less and through a one-rank NcclComm (skipped if NCCL cannot be loaded); the
random rounds are also checked against the oracle's literal ClassicPaxos instances."""
import random

import numpy as np
import pytest

from test_gpu_classic_paxos import Values, _order, splitmix64
from test_oracle_classic_paxos import CFG

pytestmark = pytest.mark.gpu

ARMS = ["local", "comm"]


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.fixture(scope="module")
def nccl(rb):
    """a one-rank NCCL communicator on device 0; None if the library cannot load NCCL"""
    try:
        import torch  # noqa: F401  (loads the libnccl.so.2 that torch ships, so the library's dlopen finds it)
        c = rb.NcclComm(0, 1, rb.NcclComm.unique_id(), 0)
    except (ImportError, rb.RapidError):
        yield None
        return
    yield c
    c.close()


@pytest.fixture(params=ARMS)
def comm(request, nccl):
    if request.param == "local":
        return None
    if nccl is None:
        pytest.skip("NCCL cannot be loaded")
    return nccl


def split(R, W, rng):
    """W contiguous, uneven, non-empty pieces of range(R) as (offset, size); with W >= 3 one of them is a single acceptor"""
    assert 1 <= W <= R
    cuts = sorted(rng.sample(range(1, R), W - 1))
    if W >= 3 and all(b - a > 1 for a, b in zip([0] + cuts, cuts + [R])):
        cuts[0] = 1                                            # a one-acceptor shard at the front
        cuts = sorted(set(cuts))
        while len(cuts) < W - 1:
            c = rng.randrange(2, R)
            if c not in cuts:
                cuts = sorted(cuts + [c])
    edges = [0] + cuts + [R]
    return [(a, b - a) for a, b in zip(edges, edges[1:])]


class Sharded:
    """one PaxosAcceptors over [begin, begin + R) and the same acceptors as W shards (listed in a shuffled order)"""

    def __init__(self, rb, cfg, R, begin, W, rng, pieces=None):
        self.whole = rb.PaxosAcceptors(cfg, R, acceptor_begin=begin)
        self.pieces = pieces or split(R, W, rng)
        self.shards = [rb.PaxosAcceptors(cfg, m, acceptor_begin=begin + o) for o, m in self.pieces]
        self.listed = list(self.shards)
        while W > 1 and self.listed == self.shards:
            rng.shuffle(self.listed)

    def register(self, acceptors, h1, ln, h2):
        acceptors = np.asarray(acceptors, np.int64)
        self.whole.registerFastRoundVotes(acceptors, h1, ln, h2)
        for (o, m), a in zip(self.pieces, self.shards):
            sel = (acceptors >= o) & (acceptors < o + m)
            if sel.any():
                a.registerFastRoundVotes(acceptors[sel] - o, np.asarray(h1)[sel], np.asarray(ln)[sel], np.asarray(h2)[sel])

    def phase1a(self, rank, msg_cfg=None):
        n = self.whole.handlePhase1aMessage(rank, msg_cfg=msg_cfg)
        self.counts = [a.handlePhase1aMessage(rank, msg_cfg=msg_cfg) for a in self.shards]
        assert sum(self.counts) == n
        return n

    def phase2a(self, rnd, value):
        n = self.whole.handlePhase2aMessage(rnd, value)
        self.counts = [a.handlePhase2aMessage(rnd, value) for a in self.shards]
        assert sum(self.counts) == n
        return n


def same1(a, b):
    assert (a.proposed, a.trigger_index, a.cval, a.n_messages) == (b.proposed, b.trigger_index, b.cval, b.n_messages), (a, b)


def same2(a, b):
    assert (a.decided, a.decided_index, a.decision) == (b.decided, b.decided_index, b.decision), (a, b)


@pytest.mark.parametrize("W", [1, 2, 3, 8])
@pytest.mark.parametrize("seed", range(4))
def test_random_rounds_match_single_handle_and_oracle(orc, rb, comm, W, seed):
    """R acceptors in W uneven shards listed out of order: 2-3 coordinators in a row on the same Paxos (its Phase1b list
    persists), then two Phase2a rounds into the same learner (its Phase2b table persists), both arrival orders"""
    rng = random.Random(900 + 31 * seed + W)
    R = rng.choice([10, 33, 128, 300])
    begin = rng.choice([0, 1000])
    u = orc.Universe()
    tags = [u.add("n", begin + r) for r in range(R)]
    hashes = [rng.randint(-50, 50) * 2 + (r % 2) for r in range(R)]
    ref = [orc.ClassicPaxos(u, tags[r], hashes[r] * 1000 + r, CFG, R) for r in range(R)]
    vals = Values()
    acc = Sharded(rb, CFG, R, begin, W, rng)
    pool = [[tags[0]], [tags[1], tags[2]], [tags[3]]]
    voters = [r for r in range(R) if rng.random() < 0.8]
    votes = {r: rng.choice(pool[: rng.randint(1, 3)]) for r in voters}
    for r, v in votes.items():
        ref[r].registerFastRoundVote(v)
    h1, h2, ln = vals.arrays([votes[r] for r in voters])
    acc.register(voters, h1, ln, h2)
    px_one, px_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    coord = ref[rng.randrange(R)]                        # the oracle's node whose Paxos both handles replay
    m2a = None
    for k in range(rng.randint(2, 3)):
        m1a = coord.startPhase1a(2 + k)
        assert px_one.startPhase1a(2 + k, m1a["rank"][1]) and px_sh.startPhase1a(2 + k, m1a["rank"][1])
        replies = {}
        for r in range(R):
            out = ref[r].handlePhase1aMessage(m1a)
            if out is not None:
                replies[begin + r] = out
        assert acc.phase1a(m1a["rank"]) == len(replies)
        perm_seed = rng.choice([0, rng.getrandbits(60) | 1])
        want = None
        for i, s in enumerate(_order(begin, sorted(replies), perm_seed)):
            out = coord.handlePhase1bMessage(replies[s])
            if out is not None:
                want = (i, out)
        one = px_one.handlePhase1bFromAcceptors(acc.whole, perm_seed)
        sh = px_sh.handlePhase1bFromAcceptorShards(acc.listed, comm=comm, perm_seed=perm_seed)
        same1(sh, one)
        if want is not None:
            assert sh.proposed and sh.trigger_index == want[0] and vals.value(sh.cval) == want[1]["vval"]
            m2a = want[1]
        else:
            assert not sh.proposed
    if m2a is None:
        return
    learner = ref[rng.randrange(R)]
    l_one, l_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    cval = vals.triple(m2a["vval"])
    for rnd in (m2a["rnd"], (10, 7)):                             # a second, higher Phase2a round into the same learner
        msg = dict(m2a, rnd=rnd)
        accepted = [begin + r for r in range(R) if ref[r].handlePhase2aMessage(msg) is not None]
        assert acc.phase2a(rnd, cval) == len(accepted)
        perm2 = rng.choice([0, rng.getrandbits(60) | 1])
        was, want2 = learner.decided(), None
        for i, s in enumerate(_order(begin, accepted, perm2)):
            if learner.handlePhase2bMessage({"sender": s - begin, "cfg": CFG, "rnd": rnd, "endpoints": m2a["vval"]}):
                want2 = i
        one = l_one.handlePhase2bFromAcceptors(acc.whole, perm2)
        sh = l_sh.handlePhase2bFromAcceptorShards(acc.listed, comm=comm, perm_seed=perm2)
        same2(sh, one)
        if not was:
            assert sh.decided == (want2 is not None)
            if want2 is not None:
                assert sh.decided_index == want2 and vals.value(sh.decision) == m2a["vval"]


def test_unpack_follows_acceptor_order_not_list_order(rb, comm):
    """the first half of the acceptors votes A, the second half B; listed second-half-first.  In acceptor order A reaches
    its N/4+1-th occurrence first — were the shards unpacked in list order, B would"""
    R = 40
    acc = Sharded(rb, CFG, R, 500, 2, random.Random(1), pieces=[(0, 20), (20, 20)])
    acc.listed = acc.shards[::-1]
    h = np.where(np.arange(R) < 20, 0xA, 0xB).astype(np.uint64)
    acc.register(np.arange(R), h, np.full(R, 2, np.int32), np.zeros(R, np.uint64))
    px_one, px_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    for p in (px_one, px_sh):
        p.startPhase1a(2, 1)
    assert acc.phase1a((2, 1)) == R
    one = px_one.handlePhase1bFromAcceptors(acc.whole)
    sh = px_sh.handlePhase1bFromAcceptorShards(acc.listed, comm=comm)
    assert one.cval == (0xA, 0, 2)
    same1(sh, one)


def test_shards_with_zero_answers(rb, comm):
    """acceptors that took a fast-round vote hold rnd (1, 1) and ignore a Phase1a / Phase2a at rank (1, 0): shards made of
    voters answer nothing while the others answer; then a round in which no shard answers at all"""
    rng = random.Random(7)
    R, begin = 60, 3
    acc = Sharded(rb, CFG, R, begin, 4, rng)
    silent = {0, 2}                                          # shards whose every acceptor voted
    voters = [o + j for i, (o, m) in enumerate(acc.pieces) if i in silent for j in range(m)]
    voters += [r for r in range(R) if rng.random() < 0.3 and r not in voters]
    voters.sort()
    h = np.array([0x55 + (r % 3) for r in voters], np.uint64)
    acc.register(voters, h, np.full(len(voters), 4, np.int32), h ^ np.uint64(0xFF))
    px_one, px_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    for p in (px_one, px_sh):
        assert p.startPhase1a(1, 0)
    assert acc.phase1a((1, 0)) == R - len(voters)
    assert [c for i, c in enumerate(acc.counts) if i in silent] == [0, 0] and sum(acc.counts) > 0
    for seed in (0, 77):                                     # the pending answers, delivered twice to the same coordinator
        same1(px_sh.handlePhase1bFromAcceptorShards(acc.listed, comm=comm, perm_seed=seed),
              px_one.handlePhase1bFromAcceptors(acc.whole, seed))
    assert acc.phase2a((1, 0), (9, 9, 1)) == R - len(voters)
    assert [c for i, c in enumerate(acc.counts) if i in silent] == [0, 0]
    l_one, l_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    same2(l_sh.handlePhase2bFromAcceptorShards(acc.listed, comm=comm, perm_seed=5), l_one.handlePhase2bFromAcceptors(acc.whole, 5))
    # nobody answers: every acceptor now holds rnd >= (1, 0), and a coordinator at (1, 0) asks again
    assert acc.phase1a((1, 0)) == 0
    px_one, px_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    for p in (px_one, px_sh):
        p.startPhase1a(1, 0)
    a, b = px_sh.handlePhase1bFromAcceptorShards(acc.listed, comm=comm), px_one.handlePhase1bFromAcceptors(acc.whole)
    same1(a, b)
    assert a.n_messages == 0 and not a.proposed
    assert acc.phase2a((1, 0), (9, 9, 1)) == 0
    same2(l_sh.handlePhase2bFromAcceptorShards(acc.listed, comm=comm), l_one.handlePhase2bFromAcceptors(acc.whole))


def test_refusals_leave_the_paxos_unchanged(rb, comm):
    """overlapping ranges, shards pending different kinds / ranks / configurations / values, a shard with nothing pending:
    each refused with EINVAL; the next valid call still gives the single-handle answer"""
    rng = random.Random(11)
    R, begin = 48, 100
    acc = Sharded(rb, CFG, R, begin, 3, rng)
    ids = np.arange(R)
    h = (ids % 2 + 1).astype(np.uint64)
    acc.register(ids, h, np.full(R, 1, np.int32), np.zeros(R, np.uint64))
    px_one, px_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    for p in (px_one, px_sh):
        p.startPhase1a(2, 4)
    assert acc.phase1a((2, 4)) == R
    past = begin + R                                         # extra handles live beyond the valid shards
    overlap = rb.PaxosAcceptors(CFG, 5, acceptor_begin=begin + acc.pieces[-1][0])
    other_rank = rb.PaxosAcceptors(CFG, 5, acceptor_begin=past)
    other_cfg = rb.PaxosAcceptors(CFG + 1, 5, acceptor_begin=past)
    other_kind = rb.PaxosAcceptors(CFG, 5, acceptor_begin=past)
    dropped = rb.PaxosAcceptors(CFG, 5, acceptor_begin=past)
    assert overlap.handlePhase1aMessage((2, 4)) == 5
    assert other_rank.handlePhase1aMessage((2, 5)) == 5
    assert other_cfg.handlePhase1aMessage((2, 4)) == 5
    assert other_kind.handlePhase2aMessage((2, 4), (1, 0, 1)) == 5
    assert dropped.handlePhase1aMessage((2, 4), msg_cfg=CFG + 9) == 0          # dropped: wrong configuration, nothing pending
    for bad in (overlap, other_rank, other_cfg, other_kind, dropped):
        with pytest.raises(rb.RapidError) as e:
            px_sh.handlePhase1bFromAcceptorShards(acc.listed + [bad], comm=comm)
        assert e.value.code == rb._native.EINVAL
    with pytest.raises(rb.RapidError) as e:
        px_sh.handlePhase1bFromAcceptorShards([], comm=comm)
    assert e.value.code == rb._native.EINVAL
    with pytest.raises(rb.RapidError) as e:
        px_sh.handlePhase2bFromAcceptorShards(acc.listed, comm=comm)          # Phase1b answers pending, not Phase2b
    assert e.value.code == rb._native.EINVAL
    one = px_one.handlePhase1bFromAcceptors(acc.whole, 3)
    same1(px_sh.handlePhase1bFromAcceptorShards(acc.listed, comm=comm, perm_seed=3), one)
    assert one.proposed
    # Phase2b: a shard that accepted a different value, or nothing, is refused; then the valid call
    assert acc.phase2a((2, 4), one.cval) == R
    other_value = rb.PaxosAcceptors(CFG, 5, acceptor_begin=past)
    assert other_value.handlePhase2aMessage((2, 4), (one.cval[0] ^ 1, one.cval[1], one.cval[2])) == 5
    l_one, l_sh = rb.Paxos(CFG, R), rb.Paxos(CFG, R)
    for bad in (other_value, other_rank, dropped):
        with pytest.raises(rb.RapidError) as e:
            l_sh.handlePhase2bFromAcceptorShards(acc.listed + [bad], comm=comm)
        assert e.value.code == rb._native.EINVAL
    same2(l_sh.handlePhase2bFromAcceptorShards(acc.listed, comm=comm, perm_seed=8), l_one.handlePhase2bFromAcceptors(acc.whole, 8))


def test_conflicting_fast_round_on_sharded_clusters(orc, rb, comm):
    """test_conflicting_fast_round_falls_back_to_classic_round with the receivers split over W VirtualCluster shards, each
    registering its votes into a PaxosAcceptors shard of the same range: the sharded Phase1b -> Phase2a on every shard ->
    sharded Phase2b reach the decision of the unsharded round"""
    from helpers import OracleWorld
    n, K, H, L = 120, 10, 9, 4
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    obs = w.tables()[0]
    cells = [(int(obs[s][r]), s, r, 1) for s in (5, 17) for r in range(K)]
    src, dst, ring, st = (np.array(x) for x in zip(*cells))
    half = np.random.default_rng(5).random(n) < 0.4
    cfg = w.view.getCurrentConfigurationId()

    def bitmap(b, m):
        bm = np.zeros((len(cells), (m + 31) // 32), np.uint32)
        for i, (_, s, _, _) in enumerate(cells):
            mask = np.ones(m, bool) if s == 5 else ~half[b: b + m]
            for r in np.nonzero(mask)[0]:
                bm[i, r // 32] |= np.uint32(1 << (r % 32))
        return bm

    whole = rb.VirtualCluster(v, H, L, kernel="bucketed")
    out = whole.handleBatch(cfg, src, dst, ring, st, bitmap=bitmap(0, n))
    acc = rb.PaxosAcceptors(cfg, n)
    acc.registerFastRoundVotesFrom(whole)
    pieces = [(0, 29), (29, 50), (79, 41)]
    shards = []
    for b, m in pieces:
        cl = rb.VirtualCluster(v, H, L, n_receivers=m, receiver_begin=b, kernel="bucketed")
        o = cl.handleBatch(cfg, src, dst, ring, st, bitmap=bitmap(b, m))
        np.testing.assert_array_equal(np.asarray(o.proposal_len), np.asarray(out.proposal_len)[b: b + m])
        a = rb.PaxosAcceptors(cfg, m, acceptor_begin=b)
        a.registerFastRoundVotesFrom(cl)
        shards.append((a, cl))
    listed = [a for a, _ in shards][::-1]
    px, px_one = rb.Paxos(cfg, n), rb.Paxos(cfg, n)
    for p in (px, px_one):
        p.startPhase1a(2, 42)
    assert acc.handlePhase1aMessage((2, 42)) == n
    assert sum(a.handlePhase1aMessage((2, 42)) for a in listed) == n
    got = px.handlePhase1bFromAcceptorShards(listed, comm=comm, perm_seed=12345)
    same1(got, px_one.handlePhase1bFromAcceptors(acc, perm_seed=12345))
    assert got.proposed and got.trigger_index == n // 2
    order = sorted(range(n), key=lambda x: (splitmix64(12345 ^ x), x))[: n // 2 + 1]
    h = np.asarray(out.proposal_hash)
    cnt, want = {}, None
    if len({int(h[r]) for r in order}) == 1:
        want = int(h[order[0]])
    else:
        for r in order:
            c = cnt.get(int(h[r]), 0)
            if c + 1 > n // 4:
                want = int(h[r])
                break
            cnt[int(h[r])] = c + 1
    assert want is not None and got.cval[0] == want
    assert acc.handlePhase2aMessage((2, 42), got.cval) == n
    assert sum(a.handlePhase2aMessage((2, 42), got.cval) for a in listed) == n
    dec = rb.Paxos(cfg, n).handlePhase2bFromAcceptorShards(listed, comm=comm, perm_seed=99)
    same2(dec, rb.Paxos(cfg, n).handlePhase2bFromAcceptors(acc, perm_seed=99))
    assert dec.decided and dec.decided_index == n // 2 and dec.decision == got.cval


def test_one_million_acceptors_in_eight_shards(rb, comm):
    """test_one_million_acceptors_classic_round's expectations with the acceptors in 8 uneven shards listed out of order,
    holding the Zipf-spread votes of test_gpu_classic_paxos_scale.py: every answer checked against tests/plainref.py, the
    Phase1b answers delivered in acceptor order and in a permuted order"""
    import plainref as P
    from test_gpu_classic_paxos_scale import zipf_votes
    n = 1_000_000
    edges = [0, 1, 90_000, 250_000, 250_001, 500_000, 640_000, 999_999, n]
    shards = [rb.PaxosAcceptors(9, b - a, acceptor_begin=a) for a, b in zip(edges, edges[1:])]
    voters, h1, h2, ln = zipf_votes(n, 8)
    ref = P.Acceptors(9, n)
    ref.registerFastRoundVotes(voters, h1, ln, h2)
    for (a, b), s in zip(zip(edges, edges[1:]), shards):
        sel = (voters >= a) & (voters < b)
        s.registerFastRoundVotes(voters[sel] - a, h1[sel], ln[sel], h2[sel])
    listed = [shards[i] for i in (5, 0, 7, 2, 6, 1, 4, 3)]
    assert sum(s.handlePhase1aMessage((2, 2)) for s in listed) == ref.phase1a((2, 2)) == n
    cval = None
    for perm in (0, 31337):
        px, coord = rb.Paxos(9, n, message_capacity=n), P.Coordinator(n, 9)
        assert px.startPhase1a(2, 2) and coord.startPhase1a(2, 2)
        got = px.handlePhase1bFromAcceptorShards(listed, comm=comm, perm_seed=perm)
        assert (got.proposed, got.trigger_index, got.cval, got.n_messages) == ref.deliver1b(coord, perm)
        assert got.proposed and got.trigger_index == n // 2 and got.n_messages == n
        cval = cval or got.cval
    assert sum(s.handlePhase2aMessage((2, 2), cval) for s in listed) == ref.phase2a((2, 2), cval) == n
    dec = rb.Paxos(9, n, message_capacity=n).handlePhase2bFromAcceptorShards(listed, comm=comm, perm_seed=4242)
    assert (dec.decided, dec.decided_index, dec.decision) == ref.deliver2b(P.Learner(n, 9), 4242)
    assert dec.decided and dec.decided_index == n // 2 and dec.decision == cval
    rng = np.random.default_rng(2)
    for r in sorted(set(rng.choice(n, size=1000, replace=False).tolist()) | {0, n - 1, 90_000, 250_000}):
        s = max(i for i, e in enumerate(edges[:-1]) if e <= r)
        assert shards[s].read(r - edges[s]) == ref.read(r), r
