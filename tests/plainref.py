"""Plain NumPy restatements of two device pieces, for the tests that check them at sizes the oracle cannot reach.

view_change   decideViewChange on a K-ring view (MembershipService.java:385-444; ringDelete / ringAdd, MembershipView.java:123-201)
              from the keys alone: which ids survive, how they are renumbered, every ring, the observer / subject tables.
FastRound     FastPaxos.handleFastRoundProposal (FastPaxos.java:125-156) over votes in arrival order, state carried across calls.

Both are pinned against the oracle by tests/test_gpu_view_change.py and tests/test_gpu_tally_cd.py (the CPU tests there)."""
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
