"""Pins the classic-Paxos pieces of tests/plainref.py (coordinator_rule, Coordinator, Learner, Acceptors) against the oracle's
literal ClassicPaxos instances (Paxos.java restated) and pyref.coordinator_rule, arrival by arrival, on random streams of a few
hundred messages.  The streams carry what the GPU tests at scale (tests/test_gpu_classic_paxos_scale.py) rely on: ranks at
INT_MIN / INT_MAX, a maximum rank held only by empty vvals, values that differ only in hash2 or only in len, pairs of values
that collide in the device's warp fold, and N such that the N/4 + 1-th occurrence falls inside the list.

Also checks, at every arrival, the fact Coordinator is built on: the rule's result is non-empty exactly when the list holds a
non-empty vval."""
import random

import numpy as np
import pytest

import plainref as P
import pyref

CFG = 1
I32_MIN, I32_MAX = -2**31, 2**31 - 1
RANKS = [(I32_MIN, I32_MIN), (I32_MIN, I32_MAX), (0, 0), (1, 1), (2, -7), (2, 7), (I32_MAX, I32_MIN), (I32_MAX, I32_MAX)]


def value_pool(n_values, seed):
    """n_values distinct (h1, h2, len) triples, built in groups of four: a fresh value, one that differs from it only in h2,
    one that differs only in len, and one whose device warp fold h1 ^ rotl(h2, 21) ^ (len << 1) equals the fresh value's"""
    k = np.arange(n_values)
    f, j = k - k % 4, k % 4
    base = P.splitmix64(f.astype(np.uint64) * np.uint64(3) + np.uint64(seed * 1_000_003))
    h1, h2 = base.copy(), P.splitmix64(base)
    lf = (f % 5 + 1).astype(np.int64)
    h2[j == 1] ^= np.uint64(1 << 40)
    ln = np.where(j == 2, lf + 7, np.where(j == 3, lf + 2, lf))
    h1 = np.where(j == 3, h1 ^ (lf << 1).astype(np.uint64) ^ (ln << 1).astype(np.uint64), h1)
    return h1, h2, ln


def fold(h1, h2, ln):
    rot = ((int(h2) << 21) | (int(h2) >> 43)) & (2**64 - 1)
    return int(h1) ^ rot ^ (int(ln) << 1)


def rule_list(rng, m, n_values, empty_top=None):
    """m Phase1b (vrnd, vval) messages in arrival order -> (vrnd (m, 2), h1, h2, len, N)"""
    top = rng.integers(2, len(RANKS))
    ranks = np.array(RANKS[: top + 1], np.int64)
    w = np.full(top + 1, 0.4 / top)
    w[top] = 0.6
    ri = rng.choice(top + 1, size=m, p=w)
    ph1, ph2, pln = value_pool(n_values, int(rng.integers(1 << 30)))
    zipf = 1.0 / np.arange(1, n_values + 1) ** 1.1
    vi = rng.choice(n_values, size=m, p=zipf / zipf.sum())
    h1, h2, ln = ph1[vi], ph2[vi], pln[vi]
    empty = rng.random(m) < 0.15
    if empty_top if empty_top is not None else rng.random() < 0.25:
        empty |= ri == top                                           # the maximum rank carries only empty vvals
    ln = np.where(empty, 0, ln)
    h1 = np.where(empty & (rng.random(m) < 0.5), h1, np.where(empty, 0, h1)).astype(np.uint64)   # len 0 is [] whatever h1 holds
    h2 = np.where(empty, 0, h2).astype(np.uint64)
    if n_values >= 4 and not (empty_top or False):
        # colliding pairs at adjacent lanes of one warp, both at the maximum rank
        k = max(1, m // 64)
        i = np.unique(rng.integers(0, max(1, m // 32), size=k) * 32 + 2 * rng.integers(0, 16, size=k))
        i = i[i + 1 < m]
        f = 4 * rng.integers(0, n_values // 4, size=len(i))
        ri[i] = ri[i + 1] = top
        h1[i], h2[i], ln[i] = ph1[f], ph2[f], pln[f]
        h1[i + 1], h2[i + 1], ln[i + 1] = ph1[f + 3], ph2[f + 3], pln[f + 3]
    vr = ranks[ri]
    col = (ri == top) & (ln > 0)
    cmax = int(np.bincount(P._value_ids(h1[col], h2[col], ln[col])).max()) if col.any() else 1
    need = int(rng.integers(1, max(2, int(cmax * 1.3) + 1)))          # N/4 + 1 inside the list, reached or not
    N = 4 * (need - 1) + int(rng.integers(0, 4))
    return vr, h1, h2, ln, max(N, 1)


class Tags:
    """(h1, h2, len) triple <-> the oracle's List<Endpoint>: one endpoint per distinct non-empty triple"""

    def __init__(self, orc):
        self.u, self.t, self.back = orc.Universe(), {}, {}

    def vval(self, h1, h2, ln):
        if ln <= 0:
            return []
        k = (int(h1), int(h2), int(ln))
        if k not in self.t:
            self.t[k] = self.u.add("v", len(self.t))
            self.back[self.t[k]] = k
        return [self.t[k]]

    def triple(self, vval):
        return None if not vval else self.back[vval[0]]


@pytest.mark.parametrize("seed", range(8))
def test_coordinator_rule_arrival_by_arrival(orc, seed):
    rng = np.random.default_rng(seed)
    m = int(rng.integers(200, 400))
    n_values = [1, 2, 5, 12, 40, 150, 300, 8][seed]
    vr, h1, h2, ln, N = rule_list(rng, m, n_values, empty_top=True if seed == 3 else None)
    tags = Tags(orc)
    msgs = [{"vrnd": (int(a), int(b)), "vval": tags.vval(x, y, z)} for (a, b), x, y, z in zip(vr, h1, h2, ln)]
    ref = orc.ClassicPaxos(tags.u, tags.u.add("me", 1), 7, CFG, N)
    for p in range(1, m + 1):
        want = ref.selectProposalUsingCoordinatorRule(msgs[:p])
        assert pyref.coordinator_rule(N, msgs[:p]) == want
        c = P.coordinator_rule(N, vr[:p], h1[:p], h2[:p], ln[:p])
        assert (tags.triple(want) if want else None) == (None if c < 0 else (int(h1[c]), int(h2[c]), int(ln[c]))), p
        assert (want != []) == bool((ln[:p] > 0).any())                  # non-empty iff a non-empty vval has arrived
        assert (c >= 0) == bool((ln[:p] > 0).any())
    assert P.coordinator_rule(N, P.pack_rank(vr), h1, h2, ln) == P.coordinator_rule(N, vr, h1, h2, ln)
    with pytest.raises(ValueError):
        P.coordinator_rule(N, vr[:0], h1[:0], h2[:0], ln[:0])


def test_value_pool_folds_collide():
    h1, h2, ln = value_pool(16, 5)
    assert len({(int(a), int(b), int(c)) for a, b, c in zip(h1, h2, ln)}) == 16
    for f in range(0, 16, 4):
        assert fold(h1[f], h2[f], ln[f]) == fold(h1[f + 3], h2[f + 3], ln[f + 3])
        assert h1[f + 1] == h1[f] and ln[f + 1] == ln[f] and h2[f + 1] != h2[f]
        assert h1[f + 2] == h1[f] and h2[f + 2] == h2[f] and ln[f + 2] != ln[f]


@pytest.mark.parametrize("seed", range(6))
def test_coordinator_across_calls(orc, seed):
    """the oracle's handlePhase1bMessage message by message vs Coordinator fed random batches and Coordinator fed one message
    per call: the trigger (call and index), cval and list size after every call; a second startPhase1a mid-stream"""
    rng = np.random.default_rng(50 + seed)
    N = int(rng.choice([5, 16, 63, 100]))
    m = int(rng.integers(200, 400))
    tags = Tags(orc)
    ref = orc.ClassicPaxos(tags.u, tags.u.add("me", 1), 77, CFG, N)
    a, b = P.Coordinator(N, CFG), P.Coordinator(N, CFG)
    assert ref.startPhase1a(2)["rank"] == (2, 77) and a.startPhase1a(2, 77) and b.startPhase1a(2, 77)
    vr, h1, h2, ln, _ = rule_list(rng, m, int(rng.choice([2, 8, 30])))
    late = seed % 2 == 1
    if late:                                                           # the first non-empty vval arrives after N/2
        ln[: min(m, N // 2 + int(rng.integers(1, 40)))] = 0
    rnd = np.where(rng.random(m) < 0.8, 0, rng.integers(1, 4, size=m))  # 0: the current crnd; others stale / higher
    cfg = np.where(rng.random(m) < 0.9, CFG, CFG + 1)
    cuts = np.sort(rng.choice(np.arange(1, m), size=6, replace=False)).tolist()
    second_at = cuts[2]
    crnd = (2, 77)
    want_total, pos = 0, 0
    for lo, hi in zip([0] + cuts, cuts + [m]):
        if lo == second_at:
            assert ref.startPhase1a(3)["rank"] == (3, 77) and a.startPhase1a(3, 77) and b.startPhase1a(3, 77)
            crnd = (3, 77)
        ranks = [crnd if r == 0 else [(2, 76), (1, 77), (3, 78)][r - 1] for r in rnd[lo:hi]]
        want = None
        for i in range(lo, hi):
            msg = {"sender": 0, "cfg": int(cfg[i]), "rnd": ranks[i - lo], "vrnd": tuple(int(x) for x in vr[i]),
                   "vval": tags.vval(h1[i], h2[i], ln[i])}
            out = ref.handlePhase1bMessage(msg)
            if out is not None:
                assert want is None
                want = (i - lo, tags.triple(out["vval"]))
            want_total += int(cfg[i] == CFG and ranks[i - lo] == crnd)
        sl = slice(lo, hi)
        got = a.handle(np.array(ranks, np.int64), vr[sl], h1[sl], ln[sl], h2[sl], msg_cfg=cfg[sl])
        assert got[3] == want_total and got[2] == tags.triple(ref.cval())
        assert (got[0], got[1]) == ((True, want[0]) if want else (False, -1))
        if want:
            assert got[2] == want[1]
        for i in range(lo, hi):                                         # one message per call
            one = b.handle(np.array([ranks[i - lo]], np.int64), vr[i:i + 1], h1[i:i + 1], ln[i:i + 1], h2[i:i + 1],
                           msg_cfg=cfg[i:i + 1])
            assert one[0] == (want is not None and want[0] == i - lo)
        assert b.cval == a.cval and b.n_messages == a.n_messages
        pos = hi
    assert pos == m


@pytest.mark.parametrize("seed", range(6))
def test_learner_across_calls(orc, seed):
    """the oracle's handlePhase2bMessage vs Learner in random batches and one message per call: repeated senders within
    and across calls, several rounds, stale configurations; the deciding message and its value"""
    rng = np.random.default_rng(80 + seed)
    N = int(rng.choice([3, 10, 41, 120]))
    m = int(rng.integers(200, 400))
    tags = Tags(orc)
    ref = orc.ClassicPaxos(tags.u, tags.u.add("me", 1), 77, CFG, N)
    a, b = P.Learner(N, CFG), P.Learner(N, CFG)
    snd = [tags.u.add("s", i) for i in range(N + 3)]
    rounds =[(2, int(x)) for x in rng.integers(-9, 9, size=int(rng.integers(1, 4)))]
    ri = rng.integers(0, len(rounds), size=m)
    sender = rng.integers(0, N + 3, size=m)
    ph1, ph2, pln = value_pool(8, seed)
    vi = rng.integers(0, 8, size=m)
    cfg = np.where(rng.random(m) < 0.9, CFG, CFG - 1)
    rk = np.array([rounds[i] for i in ri], np.int64)
    cuts = np.sort(rng.choice(np.arange(1, m), size=5, replace=False)).tolist()
    for lo, hi in zip([0] + cuts, cuts + [m]):
        want = None
        for i in range(lo, hi):
            if ref.handlePhase2bMessage({"sender": snd[sender[i]],"cfg": int(cfg[i]), "rnd": rounds[ri[i]],
                                         "endpoints": tags.vval(ph1[vi[i]], ph2[vi[i]], pln[vi[i]])}):
                assert want is None
                want = i - lo
        sl = slice(lo, hi)
        d, idx, dec = a.handle(rk[sl], sender[sl], ph1[vi[sl]], pln[vi[sl]], ph2[vi[sl]], msg_cfg=cfg[sl])
        assert d == ref.decided() and idx == (-1 if want is None else want)
        assert dec == (tags.triple(ref.decision()) if ref.decided() else None)
        for i in range(lo, hi):
            _, one, _ = b.handle(rk[i:i + 1], sender[i:i + 1], ph1[vi[i:i + 1]], pln[vi[i:i + 1]], ph2[vi[i:i + 1]],
                                 msg_cfg=cfg[i:i + 1])
            assert (one == 0) == (want == i - lo)
        assert b.decision == a.decision and b.entries == a.entries
    ok = cfg == CFG
    assert a.entries == len({(rounds[x], int(s)) for x, s in zip(ri[ok], sender[ok])}) + len({rounds[x] for x in ri[ok]})


@pytest.mark.parametrize("seed", range(4))
def test_acceptors_and_arrival_orders(orc, seed):
    """R literal instances vs Acceptors: fast-round votes with acceptors listed twice (the later vote is kept), two
    coordinators' Phase1a, Phase2a; the answers and both arrival orders, and every register"""
    rng = random.Random(seed)
    R, begin = rng.choice([7, 40, 90]), rng.choice([0, 1000])
    tags = Tags(orc)
    nodes = [tags.u.add("n", r) for r in range(R)]
    ref = [orc.ClassicPaxos(tags.u, nodes[r], 100 + r, CFG, R) for r in range(R)]
    acc = P.Acceptors(CFG, R, begin)
    ph1, ph2, pln = value_pool(8, seed)
    listed = [r for r in range(R) if rng.random() < 0.8]
    listed += rng.sample(listed, len(listed) // 4)                     # some acceptors twice, with another vote
    vi = [rng.randrange(8) for _ in listed]
    for r, v in zip(listed, vi):
        ref[r].registerFastRoundVote(tags.vval(ph1[v], ph2[v], pln[v]))
    acc.registerFastRoundVotes(listed, ph1[vi], pln[vi], ph2[vi])

    def same_registers():
        for r in range(R):
            st, rk = acc.read(r), ref[r].ranks()
            assert st["rnd"] == rk["rnd"] and st["vrnd"] == rk["vrnd"] and tags.triple(ref[r].vval()) == (
                st["vval"] if st["vval"][2] else None)

    same_registers()
    assert acc.phase1a((2, 5), msg_cfg=CFG + 1) == 0 and acc.pending is None
    for node in (5, 9):                                                # two coordinators, the second one higher
        m1a = {"sender": 0, "cfg": CFG, "rank": (2, node)}
        replies = {begin + r: out for r in range(R) if (out := ref[r].handlePhase1aMessage(m1a)) is not None}
        assert acc.phase1a((2, node)) == len(replies)
        kind, p, s, vr, h1, h2, ln = acc.pending
        assert s.tolist() == sorted(replies)
        for j, x in enumerate(s.tolist()):
            assert P.unpack_rank(vr[j]) == replies[x]["vrnd"] and tags.triple(replies[x]["vval"]) == (
                (int(h1[j]), int(h2[j]), int(ln[j])) if ln[j] else None)
        for seed2 in (0, rng.getrandbits(60) | 1):
            o = P.arrival_order(s, seed2)
            want = sorted(s.tolist(), key=lambda x: (orc.splitmix64(seed2 ^ (x & 0xFFFFFFFF)), x)) if seed2 else s.tolist()
            assert s[o].tolist() == want
        same_registers()
    v = 3
    value = (int(ph1[v]), int(ph2[v]), int(pln[v]))
    for rank in ((2, 5), (2, 9), (2, 9)):                              # rejected, accepted, then vrnd == rnd already
        m2a = {"sender": 0, "cfg": CFG, "rnd": rank, "vval": tags.vval(*value)}
        accepted = [begin + r for r in range(R) if ref[r].handlePhase2aMessage(m2a) is not None]
        assert acc.phase2a(rank, value) == len(accepted)
        assert acc.pending[2].tolist() == accepted
        same_registers()
    acc.registerFastRoundVotes(list(range(R)), ph1[:1].repeat(R), pln[:1].repeat(R), ph2[:1].repeat(R))
    for r in range(R):
        ref[r].registerFastRoundVote(tags.vval(ph1[0], ph2[0], pln[0]))  # ignored: every acceptor is in round 2
    same_registers()
