"""ClusterSimulation's graceful-leave and rejoin rules (rapid_b200/simulation.py, DESIGN.md §4.11) restated over the oracle, as a
subclass of tests/simref.py's OracleSimulation (NOT a pytest module).  OracleSimulation itself is unchanged, so every run without
leaves and rejoins is exactly the run it was.

* leave(tags): every tag must be a current member, not CRASHED, not leaving already; else ValueError and nothing changes.  In the
  next interval the leavers are CRASHED before the detectors' tick, and after the tick's and the join alerts each live entry o of
  view.getObserversOf(leaver), in ring order, adds one DOWN alert with view.getRingNumbers(o, leaver) to o's batch (one
  LeaveMessage per entry, MembershipService.leave :545-565 -> handleLeaveMessage :372-376).  A view of one member raises nothing.
* rejoin(tag, id_high, id_low): refused if the tag is a member or pending, or if the NodeId was given to this simulation before
  (creation, addJoiners, rejoin); otherwise the tag is a pending joiner again and is admitted by ringAdd with that NodeId.
* Interval records carry "leavers": the number of leavers merged in that interval."""
import numpy as np

from simref import CRASHED, DOWN, UP, OracleSimulation
from rapid_b200 import workloads as W
from rapid_b200.simulation import interval_seed


class LeaveRejoinSimulation(OracleSimulation):
    def __init__(self, orc, n, **kw):
        super().__init__(orc, n, **kw)
        self.node_id = {}                                         # joiner tag -> the NodeId it joins with
        self.seen = set(zip(*(a.tolist() for a in W.node_ids(0, n))))
        self.leaving = []

    def addJoiners(self, tags):
        for t in tags:
            self.node_id[t] = (int(self.jhi[t - self.n]), int(self.jlo[t - self.n]))
            self.seen.add(self.node_id[t])
        super().addJoiners(tags)

    def leave(self, tags):
        asked = set(self.leaving)
        for t in tags:
            if t not in self.members or self.flags[t] & CRASHED or t in asked:
                raise ValueError("tag %d cannot leave" % t)
            asked.add(t)
        self.leaving += list(tags)

    def rejoin(self, tag, id_high, id_low):
        nid = (int(id_high), int(id_low))
        if tag in self.members or tag in self.pending or nid in self.seen:
            raise ValueError("tag %d cannot rejoin with %r" % (tag, nid))
        self.node_id[tag] = nid
        self.seen.add(nid)
        self.pending.append(tag)

    def converged(self):
        return super().converged() and not self.leaving

    def interval(self):
        i, cfg = self.i, self.cfg
        leavers, self.leaving = self.leaving, []
        self.flags[leavers] = CRASHED
        batches = {}
        for o, s, rings in self.fdsim.tick(self.flags, cfg, self._edge_array()):
            batches.setdefault(o, []).append((o, s, DOWN, cfg, rings))
        if i == 0:
            for j in self.pending:                                # join phase 2: one UP alert per live expected observer
                exp = self.view.getExpectedObserversOf(j)
                for o in dict.fromkeys(exp):
                    if not self.flags[o] & CRASHED:
                        batches.setdefault(o, []).append((o, j, UP, cfg, [k for k in range(self.K) if exp[k] == o]))
        for l in leavers if self.N >= 2 else []:                  # one LeaveMessage per entry of getObserversOf
            for o in self.view.getObserversOf(l):
                if not self.flags[o] & CRASHED:
                    batches.setdefault(o, []).append((o, l, DOWN, cfg, self.view.getRingNumbers(o, l)))
        pos = {t: p for p, t in enumerate(self.members)}
        senders = sorted(batches, key=lambda o: pos[o])
        n_alerts = sum(len(batches[o]) for o in senders)
        n_cells = sum(len(m[4]) for o in senders for m in batches[o])
        rec = {"cfg": cfg, "interval": i, "alerts": n_alerts, "cells": n_cells, "announced": 0, "event": "quiet", "leavers": len(leavers)}
        decided = None
        if n_cells:
            rec["event"] = "alerts"
            blocked = np.asarray([self.flags[t] & CRASHED for t in self.ring0], np.uint8)
            ps = interval_seed(self.seed, cfg, i)
            new = []
            for b, o in enumerate(senders):
                cells = [(m[0], m[1], r, m[2]) for m in batches[o] for r in m[4]]
                src, dst, ring, st = (np.asarray(c) for c in zip(*cells))
                o_len, _, o_ids, o_off = self.sim.apply_batch(src, dst, ring, st, np.full(len(cells), cfg, np.int64), blocked=blocked,
                                                              perm_seed=ps + b, threads=4)
                for r in np.nonzero(o_len)[0]:
                    new.append((self.ring0[r], o_ids[o_off[r]: o_off[r + 1]].tolist()))
            for tag, prop in sorted(new):
                self.proposals[tag] = prop
                if self.tally.handleFastRoundProposal(tag, cfg, prop) and decided is None:
                    decided = ("fast", self.tally.decision())
            rec["announced"] = len(new)
            if new:
                rec["event"] = "proposals"
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
        self.members = [m for m in self.members if m not in set(cut)] + [t for t in self.pending if t in set(admitted)]
        self.flags[admitted] = 0
        self.pending = [t for t in self.pending if t not in set(admitted)]
        size_before, announced, votes = self.N, len(self.proposals), self.tally.votesReceived()
        self._new_configuration()
        self.history.append({"cfg_before": before, "cfg_after": self.cfg, "size_before": size_before, "size": self.N, "cut": cut,
                             "path": path, "intervals": i + 1, "announced": announced, "votes": votes,
                             "members": sorted(self.members)})
