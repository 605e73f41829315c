"""Plain NumPy restatements of device pieces, for the tests that check them at sizes the oracle cannot reach.

view_change   decideViewChange on a K-ring view (MembershipService.java:385-444; ringDelete / ringAdd, MembershipView.java:123-201)
              from the keys alone: which ids survive, how they are renumbered, every ring, the observer / subject tables.
FastRound     FastPaxos.handleFastRoundProposal (FastPaxos.java:125-156) over votes in arrival order, state carried across calls.
The classic-Paxos fallback (Paxos.java), vectorised so that 10^6 messages take seconds:
  coordinator_rule   selectProposalUsingCoordinatorRule (:271-328): the index of the message whose vval is chosen, -1 for [].
  Coordinator        the coordinator's Phase1b list, crnd and cval (:98-113, :159-191), carried across calls.
  Learner            the learner's Phase2b sets (:223-236), carried across calls.
  Acceptors          the rnd / vrnd / vval registers (:120-151, :198-216, :244-257), their compacted answers and both arrival
                     orders (acceptor order; ascending splitmix64(seed ^ uint32(sender)), ties by sender).

Coordinator relies on one fact of the rule: its result is non-empty exactly when the list holds a message with a non-empty
vval (every branch but the last picks a collected, hence non-empty, value; the last picks the first non-empty vval).  So cval
is set at the first arrival j >= N/2 (the list then holds more than N/2 messages) whose prefix holds a non-empty vval, and the
rule needs evaluating only there.  tests/test_oracle_classic_paxos_vs_plainref.py checks the fact at every arrival of random streams.

A rank (round, nodeIndex) packs into one int64 whose order is compareRanks' (signed round, then signed node index); a value
is the whole triple (h1, h2, len), len == 0 being the empty list.

view_change and FastRound are pinned against the oracle by tests/test_gpu_view_change.py and tests/test_gpu_tally_cd.py, the
classic-Paxos pieces by tests/test_oracle_classic_paxos_vs_plainref.py (the CPU tests there)."""
import numpy as np


class RingCollision(Exception):
    """two ids of the new membership share a key on some ring (the second TreeSet.add would find it)"""

    def __init__(self, ring, a, b):
        super().__init__("ring %d: new ids %d and %d share a key" % (ring, a, b))
        self.ring, self.a, self.b = ring, a, b


class ViewChange:
    __slots__ = ("old_to_new", "kept", "keys", "rings", "obs", "subj")


def view_change(keys, n, cut):
    """keys: int64 [K][tot], the ring keys of ids 0..tot-1 (members 0..n-1, then the registered joiners).  cut: ids.

    Members in the cut leave, joiners in it are admitted, the other joiners are dropped.  New ids: the surviving members in
    their old order, then the admitted joiners in id order.  Raises ValueError for an id outside [0, tot) or named twice,
    RingCollision if two new members share a key on a ring."""
    keys = np.asarray(keys, np.int64)
    K, tot = keys.shape
    cut = np.asarray(cut, np.int64)
    if len(cut) and (cut.min() < 0 or cut.max() >= tot):
        raise ValueError("cut id outside [0, %d)" % tot)
    if len(np.unique(cut)) != len(cut):
        raise ValueError("cut names an id twice")
    incut = np.zeros(tot, bool)
    incut[cut] = True
    keep = np.where(np.arange(tot) < n, ~incut, incut)
    kept = np.nonzero(keep)[0]
    n2 = len(kept)
    out = ViewChange()
    out.kept = kept
    out.old_to_new = np.full(tot, -1, np.int32)
    out.old_to_new[kept] = np.arange(n2, dtype=np.int32)
    out.keys = keys[:, kept]
    out.rings = np.argsort(out.keys, axis=1, kind="stable").astype(np.int32)       # signed int64 order
    for k in range(K):
        sk = out.keys[k, out.rings[k]]
        eq = np.nonzero(sk[1:] == sk[:-1])[0]
        if len(eq):
            raise RingCollision(k, int(out.rings[k, eq[0]]), int(out.rings[k, eq[0] + 1]))
    out.obs = np.full((n2, K), -1, np.int32)
    out.subj = np.full((n2, K), -1, np.int32)
    if n2 > 1:
        for k in range(K):
            r = out.rings[k]
            out.obs[r, k] = np.roll(r, -1)                 # successor, wrapping to the first
            out.subj[r, k] = np.roll(r, 1)                 # predecessor, wrapping to the last
    return out


def quorum(N):
    return N - (N - 1) // 4                                # FastPaxos.java:145


class FastRound:
    """The fast round of one configuration: every vote is (sender, proposal), proposal any hashable.

    sharded=False: votes are taken one by one in order; the decision is taken at the vote whose proposal's count reaches
      the quorum, and every later vote (in this call or a later one) is ignored.  count is the count at that vote,
      votes_received counts the votes up to and including it.
    sharded=True: a sharded tally has no order across ranks, so a call's votes are all counted and the decision is looked
      for at the end of the call: count and votes_received are the totals after that call."""

    def __init__(self, N, sharded=False):
        self.Q = quorum(N)
        self.sharded = sharded
        self.decided = False
        self.decision = None
        self.count = 0
        self.decided_at = None                             # (call, index in the call) of the deciding vote (in order only)
        self.calls = 0
        self.seen = set()
        self.counts = {}

    @property
    def votes_received(self):
        return len(self.seen)

    def call(self, senders, proposals):
        c = self.calls
        self.calls += 1
        if self.decided:
            return
        for i, (s, p) in enumerate(zip(senders, proposals)):
            s = int(s)
            if s in self.seen:
                continue
            self.seen.add(s)
            cnt = self.counts.get(p, 0) + 1
            self.counts[p] = cnt
            if not self.sharded and cnt >= self.Q:
                self.decided, self.decision, self.count, self.decided_at = True, p, cnt, (c, i)
                return
        if self.sharded:
            best = max(self.counts.items(), key=lambda kv: kv[1], default=(None, 0))
            if best[1] >= self.Q:
                self.decided, self.decision, self.count = True, best[0], best[1]


# ------------------------------------------------------------------------------------------------------------------ classic Paxos
_M32 = np.int64(1 << 32)


def pack_rank(rank):
    """(round, nodeIndex) pairs, shape (n, 2) or (2,) -> int64 in compareRanks order"""
    r = np.asarray(rank, np.int64)
    return r[..., 0] * _M32 + (r[..., 1] + (1 << 31))


def unpack_rank(p):
    p = int(p)
    return (p >> 32, (p & 0xFFFFFFFF) - (1 << 31))


def splitmix64(x):
    with np.errstate(over="ignore"):
        z = np.asarray(x, np.uint64) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def arrival_order(senders, perm_seed):
    """positions of `senders` in the order they arrive: as given for perm_seed 0, else ascending splitmix64(seed ^
    uint32(sender)), ties by sender"""
    s = np.asarray(senders, np.int64)
    if not perm_seed or len(s) <= 1:
        return np.arange(len(s))
    key = splitmix64(np.uint64(perm_seed & 0xFFFFFFFFFFFFFFFF) ^ (s & 0xFFFFFFFF).astype(np.uint64))
    return np.lexsort((s, key))


def _value_ids(h1, h2, ln):
    """dense ids of the distinct (h1, h2, len) triples"""
    if len(ln) == 0:
        return np.zeros(0, np.int64)
    o = np.lexsort((np.asarray(ln), np.asarray(h2), np.asarray(h1)))
    a, b, c = h1[o], h2[o], ln[o]
    new = np.ones(len(o), bool)
    new[1:] = (a[1:] != a[:-1]) | (b[1:] != b[:-1]) | (c[1:] != c[:-1])
    ids = np.empty(len(o), np.int64)
    ids[o] = np.cumsum(new) - 1
    return ids


def _kth_arrival(ids, need):
    """per id, the arrival index of its need-th occurrence (ids in arrival order); the earliest of them, or -1"""
    if need < 1 or len(ids) == 0:
        return -1
    o = np.argsort(ids, kind="stable")
    s = ids[o]
    start = np.searchsorted(s, np.arange(s[-1] + 1), side="left")
    count = np.bincount(ids)
    ok = np.nonzero(count >= need)[0]
    return int(o[start[ok] + need - 1].min()) if len(ok) else -1


def coordinator_rule(N, vrnd, h1, h2, ln):
    """selectProposalUsingCoordinatorRule over m messages in arrival order: vrnd (m, 2) ranks or packed int64, values as
    arrays.  -> index of the message whose vval is chosen, -1 for the empty list.  Raises ValueError when m == 0 (:274)."""
    ln = np.asarray(ln, np.int64)
    if len(ln) == 0:
        raise ValueError("phase1bMessages was empty")
    vr = np.asarray(vrnd, np.int64)
    vr = pack_rank(vr) if vr.ndim == 2 else vr
    h1, h2 = np.asarray(h1, np.uint64), np.asarray(h2, np.uint64)
    nonempty = np.nonzero(ln > 0)[0]
    first_nonempty = int(nonempty[0]) if len(nonempty) else -1
    col = np.nonzero((vr == vr.max()) & (ln > 0))[0]                  # collectedVvals (:278-282), arrival order
    if len(col):
        ids = _value_ids(h1[col], h2[col], ln[col])
        if ids.max() == 0:                                             # a single value (:287-289)
            return int(col[0])
        k = _kth_arrival(ids, N // 4 + 1)                              # first count + 1 > N/4 in arrival order (:293-308)
        if k >= 0:
            return int(col[k])
    return first_nonempty                                              # :319-323


class Coordinator:
    """crnd, the Phase1b list and cval of one node.  handle() takes a batch in arrival order and returns (proposed,
    trigger_index, cval, n_messages) as Paxos.handlePhase1bMessages does: trigger_index is the index in the batch of the
    message at which cval was set, cval is (h1, h2, len) or None."""

    def __init__(self, N, cfg):
        self.N, self.cfg = int(N), int(cfg)
        self.crnd = (0, 0)
        self.vr = np.zeros(0, np.int64)
        self.h1 = np.zeros(0, np.uint64)
        self.h2 = np.zeros(0, np.uint64)
        self.ln = np.zeros(0, np.int64)
        self.cval = None

    @property
    def n_messages(self):
        return len(self.ln)

    def startPhase1a(self, round_, node_index):
        """:98-113; the list is not cleared, as in the reference"""
        if self.crnd[0] > round_:
            return False
        self.crnd = (int(round_), int(node_index))
        return True

    def handle(self, rnd, vrnd, h1, ln, h2=None, msg_cfg=None):
        ln = np.asarray(ln, np.int64)
        n = len(ln)
        h2 = np.zeros(n, np.uint64) if h2 is None else np.asarray(h2, np.uint64)
        rnd, vrnd = np.asarray(rnd, np.int64), np.asarray(vrnd, np.int64)
        rnd = pack_rank(rnd) if rnd.ndim == 2 else rnd
        vrnd = pack_rank(vrnd) if vrnd.ndim == 2 else vrnd
        keep = rnd == pack_rank(self.crnd)                                 # :162-164
        if msg_cfg is not None:
            keep &= np.asarray(msg_cfg, np.int64) == self.cfg              # :157-159
        src = np.nonzero(keep)[0]
        old = self.n_messages
        self.vr = np.concatenate([self.vr, vrnd[src]])
        self.h1 = np.concatenate([self.h1, np.asarray(h1, np.uint64)[src]])
        self.h2 = np.concatenate([self.h2, h2[src]])
        self.ln = np.concatenate([self.ln, ln[src]])
        proposed, trigger = False, -1
        if self.cval is None:
            ne = np.nonzero(self.ln > 0)[0]
            if len(ne):
                j = max(self.N // 2, int(ne[0]))                       # size() > N/2 (:170) and a non-empty result
                if j < self.n_messages:
                    assert j >= old                                        # else an earlier call would have set cval
                    c = coordinator_rule(self.N, self.vr[: j + 1], self.h1[: j + 1], self.h2[: j + 1], self.ln[: j + 1])
                    self.cval = (int(self.h1[c]), int(self.h2[c]), int(self.ln[c]))          # :174-177
                    proposed, trigger = True, int(src[j - old])
        return proposed, trigger, self.cval, self.n_messages


class Learner:
    """the Phase2b sets of one node.  handle() takes a batch in arrival order and returns (decided, decided_index,
    decision) as Paxos.handlePhase2bMessages does.  entries = (rnd, sender) pairs + rounds seen, what the device's
    persistent table holds."""

    def __init__(self, N, cfg):
        self.N, self.cfg = int(N), int(cfg)
        self.rounds = {}                                                   # packed rnd -> (id, distinct senders)
        self.pairs = np.zeros(0, np.int64)                                 # sorted id << 32 | uint32(sender)
        self.decided, self.decision = False, None

    @property
    def entries(self):
        return len(self.pairs) + len(self.rounds)

    def handle(self, rnd, sender, h1, ln, h2=None, msg_cfg=None):
        ln = np.asarray(ln, np.int64)
        n = len(ln)
        h2 = np.zeros(n, np.uint64) if h2 is None else np.asarray(h2, np.uint64)
        rnd = np.asarray(rnd, np.int64)
        rnd = pack_rank(rnd) if rnd.ndim == 2 else rnd
        ok = np.ones(n, bool) if msg_cfg is None else np.asarray(msg_cfg, np.int64) == self.cfg          # :224-226
        idx = np.nonzero(ok)[0]
        ur, inv = np.unique(rnd[idx], return_inverse=True)
        for r in ur.tolist():
            self.rounds.setdefault(r, [len(self.rounds), 0])
        gid = np.array([self.rounds[r][0] for r in ur.tolist()], np.int64)[inv] if len(idx) else np.zeros(0, np.int64)
        key = (gid << 32) | (np.asarray(sender, np.int64)[idx] & 0xFFFFFFFF)
        _, first = np.unique(key, return_index=True)                        # first arrival of each pair in this call
        first = np.sort(first)
        first = first[~np.isin(key[first], self.pairs)]                     # ... that no earlier call brought
        new_idx, new_gid = idx[first], gid[first]                          # arrivals that grow their round's set (:228-230)
        decided_index = -1
        if not self.decided and len(new_idx):
            need = self.N // 2 + 1                                         # size() > N/2 (:231)
            best = None
            for r in ur.tolist():
                g, before = self.rounds[r]
                mine = new_idx[new_gid == g]
                if before < need <= before + len(mine):
                    at = int(mine[need - before - 1])
                    best = at if best is None else min(best, at)
            if best is not None:                                            # the arriving message's value (:232)
                self.decided, self.decision = True, (int(h1[best]), int(h2[best]), int(ln[best]))
                decided_index = best
        for r in ur.tolist():
            self.rounds[r][1] += int(np.count_nonzero(new_gid == self.rounds[r][0]))
        self.pairs = np.union1d(self.pairs, key[first])
        return self.decided, decided_index, self.decision


class Acceptors:
    """rnd / vrnd / vval of R acceptors; acceptor r is node begin + r.  phase1a / phase2a return the compacted answers
    (ascending sender) and keep them as `pending` for the tallies: ('1b', rank, senders, vrnd, h1, h2, len) or
    ('2b', rank, senders, value)."""

    def __init__(self, cfg, R, begin=0):
        self.cfg, self.R, self.begin = int(cfg), int(R), int(begin)
        self.rnd = np.full(R, pack_rank((0, 0)), np.int64)
        self.vrnd = self.rnd.copy()
        self.h1 = np.zeros(R, np.uint64)
        self.h2 = np.zeros(R, np.uint64)
        self.ln = np.zeros(R, np.int64)
        self.pending = None

    def registerFastRoundVotes(self, acceptor, h1, ln, h2=None):
        """:244-257 called once per listed vote in list order: an acceptor listed twice keeps its last vote"""
        a = np.asarray(acceptor, np.int64)
        if len(a) and (a.min() < 0 or a.max() >= self.R):
            raise ValueError("acceptor index out of range")
        h2 = np.zeros(len(a), np.uint64) if h2 is None else np.asarray(h2, np.uint64)
        last = len(a) - 1 - np.unique(a[::-1], return_index=True)[1]       # last listed entry of each acceptor
        last = last[(self.rnd[a[last]] >> 32) <= 1]                        # rnd.round > 1: ignored (:248-250)
        r = a[last]
        self.rnd[r] = self.vrnd[r] = pack_rank((1, 1))
        self.h1[r], self.h2[r], self.ln[r] = np.asarray(h1, np.uint64)[last], h2[last], np.asarray(ln, np.int64)[last]

    def registerFrom(self, h1, h2, ln, announced):
        """registerFastRoundVotesFrom: the receivers that announced in the last batch register their proposal"""
        a = np.nonzero(np.asarray(announced))[0]
        self.registerFastRoundVotes(a, np.asarray(h1)[a], np.asarray(ln)[a], np.asarray(h2)[a])

    def phase1a(self, rank, msg_cfg=None):
        self.pending = None
        if msg_cfg is not None and msg_cfg != self.cfg:                      # :119-121
            return 0
        p = pack_rank(rank)
        up = np.nonzero(self.rnd < p)[0]                                    # :123-125
        self.rnd[up] = p
        self.pending = ("1b", p, up + self.begin, self.vrnd[up].copy(), self.h1[up].copy(), self.h2[up].copy(), self.ln[up].copy())
        return len(up)

    def phase2a(self, rnd, value, msg_cfg=None):
        self.pending = None
        if msg_cfg is not None and msg_cfg != self.cfg:                      # :196-198
            return 0
        p = pack_rank(rnd)
        acc = np.nonzero((self.rnd <= p) & (self.vrnd != p))[0]             # :201
        self.rnd[acc] = self.vrnd[acc] = p
        self.h1[acc], self.h2[acc], self.ln[acc] = value[0], value[1], value[2]
        self.pending = ("2b", p, acc + self.begin, tuple(value))
        return len(acc)

    def deliver1b(self, coordinator, perm_seed=0):
        """the pending Phase1b answers handed to a Coordinator in arrival order"""
        kind, p, s, vr, h1, h2, ln = self.pending
        assert kind == "1b"
        o = arrival_order(s, perm_seed)
        return coordinator.handle(np.full(len(o), p, np.int64), vr[o], h1[o], ln[o], h2[o])

    def deliver2b(self, learner, perm_seed=0):
        kind, p, s, v = self.pending
        assert kind == "2b"
        o = arrival_order(s, perm_seed)
        n = len(o)
        return learner.handle(np.full(n, p, np.int64), s[o], np.full(n, v[0], np.uint64), np.full(n, v[2], np.int64),
                              np.full(n, v[1], np.uint64))

    def read(self, r):
        """-> {'rnd': (r, i), 'vrnd': (r, i), 'vval': (h1, h2, len)}, as PaxosAcceptors.read"""
        return {"rnd": unpack_rank(self.rnd[r]), "vrnd": unpack_rank(self.vrnd[r]),
                "vval": (int(self.h1[r]), int(self.h2[r]), int(self.ln[r]))}
