"""The rules of rapid_b200.simulation.ClusterSimulation restated over the oracle's literal pieces (NOT a pytest module):
FdSim for the edge detectors, join alerts built from getExpectedObserversOf, ClusterSim.apply_batch per sender batch with
the same blocked receivers and cell-order seed + b, one FastPaxosTally per configuration, ClassicPaxos instances fed in the
same arrival orders, ringDelete / ringAdd for the view change.  Node tags are the universe's tags (members 0..n-1, joiners
n..n+nj-1), which are ClusterSimulation's tags too."""
import numpy as np

from helpers import OracleWorld
from rapid_b200 import workloads as W
from rapid_b200.simulation import classic_seeds, coordinator, interval_seed

UP, DOWN = 0, 1
CRASHED = 1


class OracleSimulation:
    def __init__(self, orc, n, K=10, H=9, L=4, seed=0, n_joiners=0, fallback_intervals=1):
        self.orc, self.K, self.H, self.L, self.seed = orc, K, H, L, seed
        self.fallback_intervals = fallback_intervals
        self.w = OracleWorld(orc, n, K, n_joiners=n_joiners)
        self.view = self.w.view
        self.jhi, self.jlo = W.node_ids(n, n_joiners)
        self.n = n
        self.members = list(range(n))                             # in the device's id order
        self.flags = np.zeros(n + n_joiners, np.uint8)           # per tag
        self.edge_fail = set()
        self.pending = []
        self.history, self.intervals = [], []
        self._new_configuration()

    def setFlags(self, tag, flags):
        self.flags[tag] = flags

    def setEdgeFail(self, tag, k, fail=True):
        (self.edge_fail.add if fail else self.edge_fail.discard)((tag, k))

    def addJoiners(self, tags):
        self.pending += list(tags)

    def converged(self):
        return not self.flags[self.members].any() and not self.pending

    def _new_configuration(self):
        self.cfg = self.view.getCurrentConfigurationId()
        self.N = len(self.members)
        self.fdsim = self.orc.FdSim(self.view, self.K, np.asarray(self.members, np.int32))
        self.sim = self.orc.ClusterSim(self.view, self.K, self.H, self.L, self.N)
        self.tally = self.orc.FastPaxosTally(self.w.u, self.cfg, self.N)
        self.ring0 = list(self.view.getRing(0))
        self.proposals = {}                                       # proposer tag -> proposal (tags)
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
        batches = {}
        for o, s, rings in self.fdsim.tick(self.flags, cfg, self._edge_array()):
            batches.setdefault(o, []).append((o, s, DOWN, cfg, rings))
        if i == 0:
            for j in self.pending:                                # join phase 2: one UP alert per live expected observer
                exp = self.view.getExpectedObserversOf(j)
                for o in dict.fromkeys(exp):
                    if not self.flags[o] & CRASHED:
                        batches.setdefault(o, []).append((o, j, UP, cfg, [k for k in range(self.K) if exp[k] == o]))
        pos = {t: p for p, t in enumerate(self.members)}
        senders = sorted(batches, key=lambda o: pos[o])
        n_alerts = sum(len(batches[o]) for o in senders)
        n_cells = sum(len(m[4]) for o in senders for m in batches[o])
        rec = {"cfg": cfg, "interval": i, "alerts": n_alerts, "cells": n_cells, "announced": 0, "event": "quiet"}
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
                j = t - self.n
                self.view.ringAdd(t, (int(self.jhi[j]), int(self.jlo[j])))
                admitted.append(t)
        self.members = [m for m in self.members if m not in set(cut)] + [t for t in self.pending if t in set(admitted)]
        self.flags[admitted] = 0
        self.pending = [t for t in self.pending if t not in set(admitted)]
        size_before, announced, votes = self.N, len(self.proposals), self.tally.votesReceived()
        self._new_configuration()
        self.history.append({"cfg_before": before, "cfg_after": self.cfg, "size_before": size_before, "size": self.N, "cut": cut,
                             "path": path, "intervals": i + 1, "announced": announced, "votes": votes,
                             "members": sorted(self.members)})

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
        stuck = sorted(set(t for t in self.members if self.flags[t]) | set(self.pending))
        return {"converged": done, "stalled": not done, "intervals": total, "stuck": stuck}
