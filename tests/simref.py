"""The rules of rapid_b200.simulation.ClusterSimulation restated over the oracle's literal pieces (NOT a pytest module):
FdSim for the edge detectors, join alerts built from getExpectedObserversOf, ClusterSim.apply_batch per sender batch with
the same blocked receivers and cell-order seed + b, one FastPaxosTally per configuration, ClassicPaxos instances fed in the
same arrival orders, ringDelete / ringAdd for the view change.  Node tags are the universe's tags (members 0..n-1, joiners
n..n+nj-1), which are ClusterSimulation's tags too.

* leave(tags): every tag must be a current member, not CRASHED, not leaving already; else ValueError and nothing changes.  In the
  next interval the leavers are CRASHED before the detectors' tick, and after the tick's and the join alerts each live entry o of
  view.getObserversOf(leaver), in ring order, adds one DOWN alert with view.getRingNumbers(o, leaver) to o's batch (one
  LeaveMessage per entry, MembershipService.leave :545-565 -> handleLeaveMessage :372-376).  A view of one member raises nothing.
* rejoin(tag, id_high, id_low): refused if the tag is a member or pending, or if the NodeId was given to this simulation before
  (creation, addJoiners, rejoin); otherwise the tag is a pending joiner again and is admitted by ringAdd with that NodeId.
* batch_order "sender" hands batch b of the interval to ClusterSim.apply_batch with cell-order seed interval_seed + b;
  "shuffled" hands all of them to shuffled_ref.apply_batches with order seed interval_seed(seed, cfg, interval): every
  receiver meets the batches in its own order, the cells of a batch in array order.
* Interval records carry "leavers", the number of leavers merged in that interval, and "proposals", the number of distinct
  proposals announced in it; configuration records carry "distinct_proposals", the same over the configuration.

Below the class, the harness that drives a reference alone, or a reference and the device driver in lockstep, and compares
their runs."""
import random

import numpy as np

import shuffled_ref
from helpers import OracleWorld
from rapid_b200 import workloads as W
from rapid_b200.simulation import classic_seeds, coordinator, interval_seed

UP, DOWN = 0, 1
CRASHED = 1


class OracleSimulation:
    def __init__(self, orc, n, K=10, H=9, L=4, seed=0, n_joiners=0, fallback_intervals=1, batch_order="sender"):
        self.orc, self.K, self.H, self.L, self.seed = orc, K, H, L, seed
        self.fallback_intervals, self.batch_order = fallback_intervals, batch_order
        self.w = OracleWorld(orc, n, K, n_joiners=n_joiners)
        self.view = self.w.view
        self.jhi, self.jlo = W.node_ids(n, n_joiners)
        self.n = n
        self.tags = list(range(n))                                # the members, in the device's id order
        self.flags = np.zeros(n + n_joiners, np.uint8)           # per tag
        self.edge_fail = set()
        self.pending, self.leaving = [], []
        self.node_id = {}                                         # joiner tag -> the NodeId it joins with
        self.seen = set(zip(*(a.tolist() for a in W.node_ids(0, n))))
        self.history, self.intervals = [], []
        self._new_configuration()

    def setFlags(self, tag, flags):
        self.flags[tag] = flags

    def setEdgeFail(self, tag, k, fail=True):
        (self.edge_fail.add if fail else self.edge_fail.discard)((tag, k))

    def addJoiners(self, tags):
        for t in tags:
            self.node_id[t] = (int(self.jhi[t - self.n]), int(self.jlo[t - self.n]))
            self.seen.add(self.node_id[t])
            self.pending.append(t)

    def leave(self, tags):
        asked = set(self.leaving)
        for t in tags:
            if t not in self.tags or self.flags[t] & CRASHED or t in asked:
                raise ValueError("tag %d cannot leave" % t)
            asked.add(t)
        self.leaving += list(tags)

    def rejoin(self, tag, id_high, id_low):
        nid = (int(id_high), int(id_low))
        if tag in self.tags or tag in self.pending or nid in self.seen:
            raise ValueError("tag %d cannot rejoin with %r" % (tag, nid))
        self.node_id[tag] = nid
        self.seen.add(nid)
        self.pending.append(tag)

    def members(self):
        return list(self.tags)

    def converged(self):
        return not self.flags[self.tags].any() and not self.pending and not self.leaving

    def _new_configuration(self):
        self.cfg = self.view.getCurrentConfigurationId()
        self.N = len(self.tags)
        self.fdsim = self.orc.FdSim(self.view, self.K, np.asarray(self.tags, np.int32))
        self.sim = self.orc.ClusterSim(self.view, self.K, self.H, self.L, self.N)
        self.tally = self.orc.FastPaxosTally(self.w.u, self.cfg, self.N)
        self.ring0 = list(self.view.getRing(0))
        self.proposals = {}                                       # proposer tag -> proposal (tags)
        self.distinct = set()                                     # the configuration's proposals, as sorted tuples
        self.i = 0
        self.first_proposal = None

    def _edge_array(self):
        if not self.edge_fail:
            return None
        e = np.zeros(len(self.flags) * self.K, np.uint8)
        for t, k in self.edge_fail:
            e[t * self.K + k] = 1
        return e

    def interval(self):
        i, cfg = self.i, self.cfg
        leavers, self.leaving = self.leaving, []
        self.flags[leavers] = CRASHED
        alerts = {}                                               # sender tag -> [(sender, subject, status, rings)]
        for o, s, rings in self.fdsim.tick(self.flags, cfg, self._edge_array()):
            alerts.setdefault(o, []).append((o, s, DOWN, rings))
        if i == 0:
            for j in self.pending:                                # join phase 2: one UP alert per live expected observer
                exp = self.view.getExpectedObserversOf(j)
                for o in dict.fromkeys(exp):
                    if not self.flags[o] & CRASHED:
                        alerts.setdefault(o, []).append((o, j, UP, [k for k in range(self.K) if exp[k] == o]))
        for l in leavers if self.N >= 2 else []:                  # one LeaveMessage per entry of getObserversOf
            for o in self.view.getObserversOf(l):
                if not self.flags[o] & CRASHED:
                    alerts.setdefault(o, []).append((o, l, DOWN, self.view.getRingNumbers(o, l)))
        pos = {t: p for p, t in enumerate(self.tags)}
        senders = sorted(alerts, key=lambda o: pos[o])
        batches = [[(o, s, r, st) for o, s, st, rings in alerts[o] for r in rings] for o in senders]   # cells per sender
        rec = {"cfg": cfg, "interval": i, "alerts": sum(len(alerts[o]) for o in senders), "cells": sum(map(len, batches)),
               "announced": 0, "event": "quiet", "leavers": len(leavers), "proposals": 0}
        decided = None
        if rec["cells"]:
            rec["event"] = "alerts"
            new = self._deliver(batches, cfg, i)
            for tag, prop in sorted(new):
                self.proposals[tag] = prop
                if self.tally.handleFastRoundProposal(tag, cfg, prop) and decided is None:
                    decided = ("fast", self.tally.decision())
            rec["announced"] = len(new)
            if new:
                rec["event"] = "proposals"
                distinct = {tuple(sorted(p)) for _, p in new}
                rec["proposals"] = len(distinct)
                self.distinct |= distinct
                if self.first_proposal is None:
                    self.first_proposal = i
        if decided is None and self.first_proposal is not None and i - self.first_proposal >= self.fallback_intervals:
            value = self._classic_round(cfg, i)
            if value is None:
                rec["event"] = "stalled"
            else:
                decided = ("classic", value)
        self.i += 1
        if decided is not None:
            rec["event"] = "decided-" + decided[0]
            self._view_change(decided[0], decided[1], i)
        self.intervals.append(rec)
        return rec

    def _deliver(self, batches, cfg, i):
        """the per-sender cell batches to every live receiver -> [(receiver tag, proposal)] of the receivers that announced"""
        blocked = np.asarray([self.flags[t] & CRASHED for t in self.ring0], np.uint8)
        ps = interval_seed(self.seed, cfg, i)
        if self.batch_order == "shuffled":
            off = np.cumsum([0] + [len(b) for b in batches])
            src, dst, ring, st = (np.asarray(c) for c in zip(*(c for b in batches for c in b)))
            o_len, _, props, _ = shuffled_ref.apply_batches(self.sim, src, dst, ring, st, cfg, off, blocked=blocked, order_seed=ps)
            return [(self.ring0[r], props[r]) for r in np.nonzero(o_len)[0]]
        new = []
        for b, cells in enumerate(batches):
            src, dst, ring, st = (np.asarray(c) for c in zip(*cells))
            o_len, _, o_ids, o_off = self.sim.apply_batch(src, dst, ring, st, np.full(len(cells), cfg, np.int64), blocked=blocked,
                                                          perm_seed=ps + b, threads=4)
            new += [(self.ring0[r], o_ids[o_off[r]: o_off[r + 1]].tolist()) for r in np.nonzero(o_len)[0]]
        return new

    def _classic_round(self, cfg, i):
        orc = self.orc
        coord = coordinator(self.seed, sorted(self.proposals))
        s1, s2 = classic_seeds(self.seed, cfg, i)
        live = [r for r, t in enumerate(self.ring0) if not self.flags[t] & CRASHED]     # acceptors that answer
        px = {}
        for r in live:
            t = self.ring0[r]
            px[t] = orc.ClassicPaxos(self.w.u, t, t, cfg, self.N)
            if t in self.proposals:
                px[t].registerFastRoundVote(self.proposals[t])
        if coord not in px:                                       # a proposer that crashed since still coordinates
            px[coord] = orc.ClassicPaxos(self.w.u, coord, coord, cfg, self.N)
            px[coord].registerFastRoundVote(self.proposals[coord])
        m1a = px[coord].startPhase1a(2)

        def arrival(seed, rs):
            keys = W.splitmix64(np.asarray(rs, np.uint64) ^ np.uint64(seed))
            return [rs[j] for j in np.argsort(keys, kind="stable")]

        answers = {r: px[self.ring0[r]].handlePhase1aMessage(m1a) for r in live}
        m2a = None
        for r in arrival(s1, [r for r in live if answers[r]]):
            m2a = px[coord].handlePhase1bMessage(answers[r])
            if m2a:
                break
        if not m2a:
            return None
        accepted = {r: px[self.ring0[r]].handlePhase2aMessage(m2a) for r in live}
        for r in arrival(s2, [r for r in live if accepted[r]]):
            if px[coord].handlePhase2bMessage(accepted[r]):
                return px[coord].decision()
        return None

    def _view_change(self, path, value, i):
        cut = sorted(value)
        before = self.cfg
        admitted = []
        for t in cut:
            if self.view.isHostPresent(t):
                self.view.ringDelete(t)
            else:
                self.view.ringAdd(t, self.node_id[t])             # the NodeId of this join, a rejoin's new one included
                admitted.append(t)
        self.tags = [m for m in self.tags if m not in set(cut)] + [t for t in self.pending if t in set(admitted)]
        self.flags[admitted] = 0
        self.pending = [t for t in self.pending if t not in set(admitted)]
        size_before, announced, votes, distinct = self.N, len(self.proposals), self.tally.votesReceived(), len(self.distinct)
        self._new_configuration()
        self.history.append({"cfg_before": before, "cfg_after": self.cfg, "size_before": size_before, "size": self.N, "cut": cut,
                             "path": path, "intervals": i + 1, "announced": announced, "votes": votes,
                             "members": sorted(self.tags), "distinct_proposals": distinct})

    def run(self, max_intervals):
        since, total = 0, 0
        while not self.converged():
            if since >= max_intervals:
                break
            rec = self.interval()
            total += 1
            since = 0 if rec["event"].startswith("decided") else since + 1
            if rec["event"] == "stalled":
                break
        done = self.converged()
        stuck = sorted(set(t for t in self.tags if self.flags[t]) | set(self.pending))
        return {"converged": done, "stalled": not done, "intervals": total, "stuck": stuck}


# ---- lockstep: every call applied to a reference alone, or to a reference and the device driver ------------------------------
def make(orc, rb, n, seed, n_joiners=0, **kw):
    """(reference,) or, given the package rb, (reference, driver): members 0..n-1; joiners n..n+n_joiners-1 are known to the
    reference and ask to join by join().  The keywords (batch_order, ...) go to both."""
    sims = [OracleSimulation(orc, n, seed=seed, n_joiners=n_joiners, **kw)]
    if rb is not None:
        sims.append(rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed, **kw))
    return tuple(sims)


def join(sims, tags):
    """the next joiner tags, consecutive, ask to join (the two addJoiners take different arguments)"""
    tags = list(tags)
    for s in sims:
        if isinstance(s, OracleSimulation):
            s.addJoiners(tags)
        elif tags:
            assert s.addJoiners(*W.endpoints(tags[0], len(tags)), *W.node_ids(tags[0], len(tags))) == tags


def flags(sims, tags, f):
    for s in sims:
        for t in tags:
            s.setFlags(t, f)


def leave(sims, tags):
    for s in sims:
        s.leave(tags)


def rejoin(sims, tag, node_id):
    for s in sims:
        s.rejoin(tag, *node_id)


def run(sims, max_intervals=30):
    """every simulation runs to convergence -> the first one's run()"""
    outs = [s.run(max_intervals) for s in sims]
    assert all(o["converged"] for o in outs), outs
    return outs[0]


def steps(sims, count):
    """count intervals of every simulation -> the first one's records"""
    return [[s.interval() for s in sims][0] for _ in range(count)]


def random_hosts(n, count, seed, lo=0):
    return sorted(random.Random(seed).sample(range(lo, n), count))


def same_run(ref, dev):
    """every key of every interval and configuration record the reference wrote is equal in the driver's records (which add
    their timings), and the memberships are equal"""
    for mine, theirs in ((ref.intervals, dev.intervals), (ref.history, dev.history)):
        assert len(theirs) == len(mine)
        assert [{k: d[k] for k in r} for r, d in zip(mine, theirs)] == mine
    assert sorted(dev.members()) == sorted(ref.members())
