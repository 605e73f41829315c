"""ClusterSimulation(batch_order=...) restated over the oracle (NOT a pytest module): a subclass of tests/simref_leave.py's
LeaveRejoinSimulation (which extends tests/simref.py; both unchanged) whose step 3 hands the interval's sender batches to
shuffled_ref.apply_batches with order seed interval_seed(seed, cfg, interval) when batch_order == "shuffled" (every receiver
meets the batches in its own order, cells of a batch in array order), and to ClusterSim.apply_batch with cell-order seed + b, as
simref does, when batch_order == "sender".  It also keeps the two record keys of the device driver: intervals[i]["proposals"],
the number of distinct proposals announced in the interval, and history[c]["distinct_proposals"], the same over the
configuration."""
import numpy as np

import shuffled_ref
from simref import CRASHED, DOWN, UP
from simref_leave import LeaveRejoinSimulation
from rapid_b200.simulation import interval_seed


class ShuffledSimulation(LeaveRejoinSimulation):
    def __init__(self, orc, n, batch_order="sender", **kw):
        self.batch_order = batch_order
        super().__init__(orc, n, **kw)

    def _new_configuration(self):
        super()._new_configuration()
        self.distinct = set()

    def _deliver(self, senders, batches, cfg, i):
        """step 3 -> [(receiver tag, proposal)] of the receivers that announced"""
        blocked = np.asarray([self.flags[t] & CRASHED for t in self.ring0], np.uint8)
        ps = interval_seed(self.seed, cfg, i)
        new = []
        if self.batch_order == "shuffled":
            cells = [(m[0], m[1], r, m[2]) for o in senders for m in batches[o] for r in m[4]]
            off = np.cumsum([0] + [sum(len(m[4]) for m in batches[o]) for o in senders])
            src, dst, ring, st = (np.asarray(c) for c in zip(*cells))
            o_len, _, props, _ = shuffled_ref.apply_batches(self.sim, src, dst, ring, st, cfg, off, blocked=blocked, order_seed=ps)
            return [(self.ring0[r], props[r]) for r in np.nonzero(o_len)[0]]
        for b, o in enumerate(senders):
            cells = [(m[0], m[1], r, m[2]) for m in batches[o] for r in m[4]]
            src, dst, ring, st = (np.asarray(c) for c in zip(*cells))
            o_len, _, o_ids, o_off = self.sim.apply_batch(src, dst, ring, st, np.full(len(cells), cfg, np.int64), blocked=blocked,
                                                          perm_seed=ps + b, threads=4)
            for r in np.nonzero(o_len)[0]:
                new.append((self.ring0[r], o_ids[o_off[r]: o_off[r + 1]].tolist()))
        return new

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
        rec = {"cfg": cfg, "interval": i, "alerts": n_alerts, "cells": n_cells, "announced": 0, "event": "quiet", "leavers": len(leavers),
               "proposals": 0}
        decided = None
        if n_cells:
            rec["event"] = "alerts"
            new = self._deliver(senders, batches, cfg, i)
            for tag, prop in sorted(new):
                self.proposals[tag] = prop
                if self.tally.handleFastRoundProposal(tag, cfg, prop) and decided is None:
                    decided = ("fast", self.tally.decision())
            rec["announced"] = len(new)
            if new:
                rec["event"] = "proposals"
                rec["proposals"] = len({tuple(sorted(p)) for _, p in new})
                self.distinct |= {tuple(sorted(p)) for _, p in new}
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
        distinct = len(self.distinct)
        super()._view_change(path, value, i)
        self.history[-1]["distinct_proposals"] = distinct
