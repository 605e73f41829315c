"""A whole Rapid cluster simulated on the device, configuration after configuration: the loop MembershipService runs
(alert generation -> per-sender alert batches -> cut detection -> fast round -> classic fallback -> decideViewChange,
MembershipService.java:300-354, :385-444, FastPaxos.java:94-203), composed from the classes of this package.

ClusterSimulation rules (tests/simref.py restates them independently; DESIGN.md §4.11):

* Nodes are named by TAGS: the members given at creation are 0..n-1 in the given order, joiners get the next tags in the
  order addJoiners() lists them.  Tags never change; the device ids of a configuration are dense (view.applyCut renumbers),
  and the driver keeps the id -> tag map.  Scenario flags (failure_detector.CRASHED, INGRESS_BLOCKED, ...) are kept per tag,
  so a view change carries them over; an admitted joiner starts with flags 0.
* One interval, in this order:
    0. the members that asked to leave since the last interval (leave()) get the CRASHED flag: they have shut down, so they
       answer no probe, run no detector, receive nothing, and their acceptors are silent;
    1. one failure-detector interval of every member (EdgeFailureDetectors.tickDevice with the members' flags);
    2. one merge into that interval (mergeAlerts): in the FIRST interval of a configuration only, every pending joiner asks
       again (one join attempt per configuration: its live expected observers each send one UP alert); and every leaver of
       step 0 sends its LeaveMessages (MembershipService.leave :545-565): each live entry o of getObserversOf(leaver) raises
       one DOWN alert with getRingNumbers(o, leaver), repeats kept (handleLeaveMessage :372-376);
    3. the interval's alerts, one batch per sender in ascending sender id, reach every receiver (receiver r = ring-0
       position r) through VirtualCluster.handleBatchesDevice: crashed receivers get nothing, batch b reaches receiver r in
       its own cell order seeded interval_seed(seed, cfg, interval) + b;
    4. every receiver that announced registers its fast-round vote with its acceptor (FastPaxos.propose :94-98);
    5. one FastPaxos tally of those votes; the tally accumulates over the configuration's intervals.
  Steps 3-5 are skipped in an interval without alerts.
* Fallback: if the fast round has not decided at the end of interval i0 + fallback_intervals (i0 = the configuration's
  first interval with a proposal), the classic round runs in that interval: the coordinator is the proposer with the
  smallest splitmix64(seed ^ tag) (a seeded stand-in for the expovariate jitter of FastPaxos.java:200-203); its
  Phase1a has rank (2, coordinator tag); crashed acceptors are silent; Phase1b and Phase2b answers arrive in ascending
  splitmix64(phase_seed ^ ring-0 position) order (phase_seed = classic_seeds(...)).  A classic round that does not decide
  stalls the run.
* View change (decideViewChange :385-444): a proposer of the decided value is found on the device
  (PaxosAcceptors.findValue, before any Phase2a), its proposal is the cut; view.applyCut; joiners not admitted are
  registered again with their NodeIds; the configuration id comes from the device's identifiersSeen; the detectors are
  reset; the cut detector and the acceptors are created anew for the new membership size.
* Leave (leave(tags)): every tag must be a current member that is not CRASHED and has not asked to leave already, else
  ValueError and nothing changes.  A leave is one-shot, as in the reference: if the interval's decision does not include a
  leaver, it stays a crashed member and the detectors cut it later.  Interval records count the leavers merged ("leavers").
* Rejoin (rejoin(tag, id_high, id_low)): the endpoint of a departed tag asks to join again with a new NodeId, as the same tag
  (tags name endpoints).  Refused with ValueError and no change if the tag is still a member (HOSTNAME_ALREADY_IN_RING), is
  already pending, or if the NodeId was ever given to this simulation (UUID_ALREADY_IN_RING: creation, addJoiners, rejoin).
  Otherwise the tag becomes a pending joiner under the join rules above, and its flags are cleared on admission.
* Delivery model (batch_order): with "sender" (the default) every receiver gets the senders' batches in the same (ascending
  sender) order and only the cell order within a batch is per receiver, as step 3 says.  With "shuffled" every receiver meets the
  interval's batches in its own pseudo-random order, as the reference's per-sender shuffled recipient lists make it
  (UnicastToAllBroadcaster.java:59-62), and the cells of each batch in array order (one message is parsed in one order): the
  configuration's VirtualCluster is a sweep handle and step 3 passes batch_order_seed = interval_seed(seed, cfg, interval)
  (RAPID_DELIVERY_SHUFFLED_BATCHES) instead of the cell-order seeds.  Nothing else in the interval changes.  Receivers that
  meet the batches in different orders can announce different proposals; the records count them: intervals[i]["proposals"]
  is the number of distinct proposals announced in the interval, history[c]["distinct_proposals"] the number over the
  configuration.  Every node sees every vote, so one tally stands for every node's.
* Wire traffic (wire_traffic=True; off by default, and then no record changes): every interval record gains wire_bytes, the
  bytes of the interval's alert batches, fast-round votes and (when a classic round ran) Phase1b / Phase2b answers, each wrapped
  as a RapidRequest, encoded on the device and counted once per member (a broadcast is one unicast per member,
  UnicastToAllBroadcaster.java:46-52); wire_tx_max / wire_tx_mean over the members' transmitted bytes and wire_rx_max /
  wire_rx_mean (every member receives every broadcast, so they are equal).  Probes, join messages and LeaveMessage are not
  encoded: these are not the traffic figures of the Rapid paper.
* Overlay quality (overlay_quality=True; off by default, and then no record changes): every configuration record gains
  overlay_ratio and overlay_residual, MembershipView.overlaySpectrum() (default seed, tolerance and step limit) of the view
  AFTER that view change: lambda / 2K of its monitoring overlay and the bound on the error of lambda (DESIGN.md §4.13);
  initial_overlay holds the same pair for the view the simulation started with.  Both are None for a view of fewer than 3
  members, which has no such figure.
* Proposal census (proposal_census=True; off by default, and then no record changes): every interval record with announcers
  gains census, the distinct proposals announced in that interval (VirtualCluster.proposalCensus, counted on the device) in
  order of their lowest announcing receiver, each {"size", "down", "up", "voters", "representative"}: its length, its
  entries that are members (DOWN) and registered joiners (UP) as VIEW_CHANGE_PROPOSAL lists them, how many receivers announced
  it, and the tag of the lowest of them.  Every configuration record gains census, the interval censuses merged by proposal
  in order of first appearance, each {"size", "down", "up", "voters", "decided", "missing", "extra"}: decided marks the
  decided cut, missing / extra count the cut's nodes the proposal lacks and the nodes it names outside the cut; and agreement,
  the decided proposal's voters over the configuration's announcers.
"""
import time

import numpy as np

from . import _native as N
from .classic_paxos import Paxos, PaxosAcceptors
from .cut_detector import VirtualCluster
from .failure_detector import CRASHED, EdgeFailureDetectors, FAILURE_THRESHOLD
from .fast_paxos import FastPaxos
from .membership_view import MembershipView
from .wire import WireDecoder
from .workloads import splitmix64

_M64 = 0xFFFFFFFFFFFFFFFF


def _sm(x):
    return int(splitmix64(np.uint64(x & _M64)))


def interval_seed(seed, cfg, interval):
    """cell-order seed of one interval: batch b of it is delivered with interval_seed + b"""
    return _sm(_sm(seed ^ cfg) + interval)


def classic_seeds(seed, cfg, interval):
    """(Phase1b, Phase2b) arrival-order seeds of a classic round run in that interval (never 0: 0 means acceptor order)"""
    s = interval_seed(seed, cfg, interval)
    return _sm(s ^ 1) or 1, _sm(s ^ 2) or 1


def coordinator(seed, proposer_tags):
    """the proposer whose recovery timer fires first: smallest splitmix64(seed ^ tag), ties by tag"""
    t = np.asarray(proposer_tags, np.uint64)
    keys = splitmix64(t ^ np.uint64(seed & _M64))
    return int(t[np.lexsort((t, keys))[0]])


class ClusterSimulation:
    """ClusterSimulation((host_bytes, host_off, ports), (id_high, id_low)): a cluster of the given members on one device.

    setFlags / setEdgeFail / addJoiners / leave / rejoin describe the scenario; interval() runs one failure-detector interval of the whole
    cluster; run() runs intervals until the membership has converged or the run stalls.  history holds one record per
    configuration, intervals one per interval."""

    def __init__(self, endpoints, node_ids, K=10, H=9, L=4, seed=0, failure_threshold=FAILURE_THRESHOLD, fallback_intervals=1,
                 device=0, batch_order="sender", overlay_quality=False, wire_traffic=False, proposal_census=False):
        if batch_order not in ("sender", "shuffled"):
            raise ValueError("batch_order is 'sender' or 'shuffled', not %r" % (batch_order,))
        self.batch_order = batch_order
        import torch                                              # device buffers of the scenario's flags
        self._torch = torch
        self.K, self.H, self.L, self.seed, self.device = int(K), int(H), int(L), int(seed), device
        self.fallback_intervals = int(fallback_intervals)
        self.proposal_census = bool(proposal_census)
        hb, off, ports = endpoints
        self.view = MembershipView.from_packed(self.K, hb, off, ports, device=device)
        self.view.setNodeIds(*node_ids)
        n = len(ports)
        # creation endpoints per tag, so that a departed member can register its hostname and port again (rejoin)
        self._hb, self._off, self._ports = (np.array(a, copy=True) for a in (hb, off, ports))
        self._seen_hi, self._seen_lo, self._n_seen = np.zeros(0, np.int64), np.zeros(0, np.int64), 0
        self._add_seen(node_ids[0], node_ids[1])                  # every NodeId this simulation was given, as arrays
        self.leaving = []                                         # tags that leave in the next interval, in call order
        self.tags = np.arange(n, dtype=np.int64)                  # device id -> tag
        self.flags = np.zeros(n, np.uint8)                        # per tag
        self.edge_fail = {}                                       # (tag, k) -> probes of that tag's k-th detector fail
        self.joiners = {}                                         # tag -> (hostname, port, id_high, id_low)
        self.pending = []                                         # joiner tags not yet admitted, in tag order
        self.history, self.intervals = [], []
        self.cfg = self.view.currentConfigurationId()
        self.fd = EdgeFailureDetectors(self.view, failure_threshold)
        self.fp = None
        self._new_handles()
        self.overlay_quality = bool(overlay_quality)
        self.initial_overlay = self._overlay() if self.overlay_quality else None
        self.wire = WireDecoder(self.view) if wire_traffic else None     # sizes of the interval's messages, encoded on the device
        self._wire_tx = None

    # ---- scenario ------------------------------------------------------------------------------------------------------------
    def setFlags(self, node, flags):
        """RAPID_FD_* bits of a node (tag); applies from the next interval"""
        self.flags[int(node)] = np.uint8(flags)
        self._dirty = True

    def setEdgeFail(self, node, k, fail=True):
        """probes of node's k-th detector (k-th entry of getSubjectsOf, current configuration) fail regardless of flags"""
        if fail:
            self.edge_fail[(int(node), int(k))] = True
        else:
            self.edge_fail.pop((int(node), int(k)), None)
        self._dirty = True

    def addJoiners(self, hostnames, ports, id_high, id_low):
        """endpoints that ask to join from the next configuration's first interval on (the current one if it has not run an
        interval yet); -> their tags"""
        first = len(self.flags)
        tags = list(range(first, first + len(ports)))
        for i, t in enumerate(tags):
            self.joiners[t] = (hostnames[i], int(ports[i]), int(id_high[i]), int(id_low[i]))
        self._add_seen(id_high, id_low)
        self.flags = np.concatenate([self.flags, np.zeros(len(tags), np.uint8)])
        self._register(tags)
        self.pending += tags
        return tags

    def leave(self, tags):
        """Cluster.leaveGracefully of each tag: in the next interval the tags shut down (CRASHED) and their observers raise
        the leave alerts in that interval's merge"""
        tags = [int(t) for t in tags]
        member = np.zeros(len(self.flags), bool)
        member[self.tags] = True
        asked = set(self.leaving)
        for t in tags:
            if not 0 <= t < len(self.flags) or not member[t]:
                raise ValueError("tag %d is not a member" % t)
            if self.flags[t] & CRASHED:
                raise ValueError("tag %d has crashed" % t)
            if t in asked:
                raise ValueError("tag %d is leaving already" % t)
            asked.add(t)
        self.leaving += tags

    def rejoin(self, tag, id_high, id_low):
        """the endpoint of departed tag asks to join again with NodeId (id_high, id_low), from the next configuration's first
        interval on (the current one if it has not run an interval yet)"""
        t, hi, lo = int(tag), int(id_high), int(id_low)
        if not 0 <= t < len(self.flags):
            raise ValueError("tag %d names no endpoint of this simulation" % t)
        if (self.tags == t).any():
            raise ValueError("tag %d is a member (HOSTNAME_ALREADY_IN_RING)" % t)
        if t in self.pending:
            raise ValueError("tag %d is already asking to join" % t)
        k = self._n_seen
        if ((self._seen_hi[:k] == hi) & (self._seen_lo[:k] == lo)).any():
            raise ValueError("NodeId of tag %d was seen before (UUID_ALREADY_IN_RING)" % t)
        if t in self.joiners:
            host, port = self.joiners[t][:2]
        else:
            host, port = self._hb[self._off[t]: self._off[t + 1]].tobytes(), int(self._ports[t])
        self.joiners[t] = (host, port, hi, lo)
        self._add_seen([hi], [lo])
        self._register([t])
        self.pending.append(t)

    def members(self):
        """tags of the current members, in device id order"""
        return self.tags.tolist()

    def converged(self):
        return not self.flags[self.tags].any() and not self.pending and not self.leaving

    def _add_seen(self, id_high, id_low):
        hi, lo = np.asarray(id_high, np.int64), np.asarray(id_low, np.int64)
        k, m = self._n_seen, len(hi)
        if k + m > len(self._seen_hi):                            # doubling: a rejoin appends one id
            cap = max(2 * len(self._seen_hi), k + m, 16)
            self._seen_hi = np.concatenate([self._seen_hi[:k], np.zeros(cap - k, np.int64)])
            self._seen_lo = np.concatenate([self._seen_lo[:k], np.zeros(cap - k, np.int64)])
        self._seen_hi[k: k + m], self._seen_lo[k: k + m] = hi, lo
        self._n_seen = k + m

    # ---- handles of one configuration ------------------------------------------------------------------------------------------
    def _register(self, tags):
        if not tags:
            return
        ids = self.view.registerJoiners([self.joiners[t][0] for t in tags], [self.joiners[t][1] for t in tags])
        self.view.setJoinerIds(ids[0], [self.joiners[t][2] for t in tags], [self.joiners[t][3] for t in tags])
        self.joiner_id.update(zip(tags, ids))

    def _new_handles(self):
        n = self.view.n
        self.N = n
        self.cl = VirtualCluster(self.view, self.H, self.L, kernel="sweep" if self.batch_order == "shuffled" else "bucketed")
        self.acc = PaxosAcceptors(self.cfg, n, device=self.device)
        if self.fp is None or n > self._fp_cap:
            self.fp, self._fp_cap = FastPaxos(self.cfg, n, device=self.device), n
        else:
            self.fp.reset(self.cfg, n)
        self.ring0 = np.asarray(self.view.getRing(0), np.int64)
        self.joiner_id = {}
        self.interval_in_cfg = 0
        self.first_proposal = None
        self.votes = 0
        self.announced = 0
        self.proposal_fps = set()                                 # (h1, h2, len) of every proposal announced in the configuration
        self.census = {}                                          # proposal_census: (h1, h2, len) -> the configuration's class
        self._census_interval = None                              # ... and the interval of the cluster's last census
        self._ann = None                                          # announcedProposal flags, read at most once per interval
        self._dirty = True
        self._cfg_t = {"detect_ms": 0.0, "classic_ms": 0.0, "view_change_ms": 0.0, "handles_ms": 0.0, "device_ms": 0.0}

    def _upload_flags(self):
        torch = self._torch
        f = self.flags[self.tags]
        self.d_flags = torch.from_numpy(np.ascontiguousarray(f)).to("cuda:%d" % self.device)
        self.crashed_r = (f[self.ring0] & CRASHED) != 0                  # per receiver / acceptor
        self.d_blocked = torch.from_numpy(self.crashed_r.astype(np.uint8)).to("cuda:%d" % self.device)
        self.d_edge = None
        if self.edge_fail:
            pos = {int(t): i for i, t in enumerate(self.tags)}
            e = np.zeros(self.N * self.K, np.uint8)
            for (t, k) in self.edge_fail:
                if t in pos:
                    e[pos[t] * self.K + k] = 1
            self.d_edge = torch.from_numpy(e).to("cuda:%d" % self.device)
        self._dirty = False

    # ---- one interval ----------------------------------------------------------------------------------------------------------
    def interval(self):
        """one failure-detector interval of the cluster -> its record (also appended to intervals); record["event"] is
        quiet / alerts / proposals / decided-fast / decided-classic (the view has changed) / stalled"""
        t0 = time.perf_counter()
        self._ann = None
        leavers, self.leaving = self.leaving, []
        if leavers:
            self.flags[leavers] = CRASHED                         # shut down: silent from this interval on
            self._dirty = True
        if self._dirty:
            self._upload_flags()
        i, cfg = self.interval_in_cfg, self.cfg
        na, nc = self.fd.tickDevice(self.d_flags.data_ptr(), cfg, 0 if self.d_edge is None else self.d_edge.data_ptr())
        dev_ms = self.fd.lastDeviceMs()
        joiners = [self.joiner_id[t] for t in self.pending] if i == 0 else []
        if joiners or leavers:
            na, nc = self.fd.mergeAlerts(joiners, self._member_ids(leavers), cfg)
            dev_ms += self.fd.lastDeviceMs()
        rec = {"cfg": cfg, "interval": i, "alerts": na, "cells": nc, "announced": 0, "event": "quiet", "leavers": len(leavers),
               "proposals": 0}
        decided = None
        n_members = self.N
        if self.wire is not None:
            self._wire_tx = np.zeros(n_members, np.float64)
            if na:
                self._wire_count(lambda: N.check(N.lib().rapid_wire_encode_alert_batches(self.wire._h, self.fd._h, N.WIRE_REQUEST, None, None)))
        if nc:
            rec["event"] = "alerts"
            p = self.fd.cellsDevice()
            order = {"batch_order_seed" if self.batch_order == "shuffled" else "perm_seed": interval_seed(self.seed, cfg, i)}
            self.cl.handleBatchesDevice(cfg, nc, p[1], p[2], p[3], self.fd.senderBatches(), cell_cfg_dev=p[4],
                                        blocked_dev=self.d_blocked.data_ptr(), **order)
            dev_ms += self.cl.lastDeviceMs()[0]
            self.acc.registerFastRoundVotesFrom(self.cl)
            if self.wire is not None:
                self._wire_count(lambda: N.check(N.lib().rapid_wire_encode_votes(self.wire._h, self.cl._h, cfg, N.WIRE_REQUEST, None,
                                                                                 None)))
            t = self.fp.tallyCluster(self.cl)
            dev_ms += self.fp.lastDeviceMs()
            # votes are counted up to the decision (FastPaxos.java:138): in a deciding interval the announcers are counted instead,
            # from the announcedProposal flags (1 B per receiver, read once per configuration)
            rec["announced"] = int(self._announced_flags().sum()) - self.announced if t.decided else t.votes_received - self.votes
            self.votes = t.votes_received
            if rec["announced"]:
                out = self.cl.readOutputs()                       # the proposals announced in this interval
                now = out.proposal_len > 0
                fps = set(zip(out.proposal_hash[now].tolist(), out.proposal_hash2[now].tolist(), out.proposal_len[now].tolist()))
                rec["proposals"] = len(fps)
                self.proposal_fps |= fps
                rec["event"] = "proposals"
                if self.proposal_census:
                    rec["census"] = self._interval_census(i)
                self.announced += rec["announced"]
                if self.first_proposal is None:
                    self.first_proposal = i
            if t.decided:
                decided = ("fast", (t.hash, t.hash2, t.length))
        self._cfg_t["detect_ms"] += (time.perf_counter() - t0) * 1e3
        if decided is None and self.first_proposal is not None and i - self.first_proposal >= self.fallback_intervals:
            t1 = time.perf_counter()
            value, ms = self._classic_round(cfg, i)
            self._cfg_t["classic_ms"] += (time.perf_counter() - t1) * 1e3
            dev_ms += ms
            if value is None:
                rec["event"] = "stalled"
            else:
                decided = ("classic", value)
        if self.wire is not None:
            # a broadcast is one unicast per member (UnicastToAllBroadcaster.java:46-52): every member receives every message
            tx = self._wire_tx
            rec["wire_bytes"] = int(tx.sum())
            rec["wire_tx_max"], rec["wire_tx_mean"] = int(tx.max()), float(tx.mean())
            rx = rec["wire_bytes"] // n_members
            rec["wire_rx_max"], rec["wire_rx_mean"] = rx, float(rx)
        self._cfg_t["device_ms"] += dev_ms
        rec["device_ms"] = dev_ms
        rec["host_ms"] = (time.perf_counter() - t0) * 1e3               # host clock of the whole interval, view change excluded
        self.interval_in_cfg += 1
        if decided is not None:
            rec["event"] = "decided-" + decided[0]
            self._view_change(decided[0], decided[1], i)
        self.intervals.append(rec)
        return rec

    def _member_ids(self, tags):
        """device ids of member tags"""
        if not tags:
            return []
        inv = np.full(len(self.flags), -1, np.int64)
        inv[self.tags] = np.arange(len(self.tags))
        return inv[np.asarray(tags, np.int64)]

    def _classic_round(self, cfg, i):
        """Paxos.java round 2 from the seeded coordinator over the acceptors -> (decided value or None, device ms)"""
        ann = self._announced_flags() != 0
        coord = coordinator(self.seed, self.tags[self.ring0[ann]])
        s1, s2 = classic_seeds(self.seed, cfg, i)
        px = Paxos(cfg, self.N, device=self.device)
        try:
            return self._rounds(px, coord, s1, s2)
        finally:
            px.close()

    def _rounds(self, px, coord, s1, s2):
        px.startPhase1a(2, coord)
        self.acc.setSilent(self.crashed_r)
        self.acc.handlePhase1aMessage((2, coord))
        if self.wire is not None:
            self._wire_count(lambda: N.check(N.lib().rapid_wire_encode_phase1b(self.wire._h, self.acc._h, self.cl._h, N.WIRE_REQUEST,
                                                                               None, None)))
        r1 = px.handlePhase1bFromAcceptors(self.acc, perm_seed=s1)
        ms = px.lastDeviceMs()
        if not r1.proposed:
            return None, ms
        self._proposer = self.acc.findValue(r1.cval)                # before Phase2a overwrites the vvals
        self.acc.handlePhase2aMessage((2, coord), r1.cval)
        if self.wire is not None:
            self._wire_count(lambda: N.check(N.lib().rapid_wire_encode_phase2b(self.wire._h, self.acc._h, self.cl._h, N.WIRE_REQUEST,
                                                                               None, None)))
        r2 = px.handlePhase2bFromAcceptors(self.acc, perm_seed=s2)
        ms += px.lastDeviceMs()
        return (r2.decision if r2.decided else None), ms

    def _wire_count(self, encode):
        """encode one kind of the interval's messages on the device (wrapped as RapidRequests) and add size x members to each
        sender's transmitted bytes; only the sizes and senders leave the device"""
        encode()
        sizes, senders = self.wire.encodedSizes(), self.wire.encodedSenders()
        if len(sizes):
            self._wire_tx += np.bincount(senders, weights=sizes.astype(np.float64) * self.N, minlength=self.N)[: self.N]

    def _interval_census(self, i):
        """the interval's census record; its classes are merged into the configuration's by fingerprint"""
        c = self.cl.proposalCensus()
        self._census_interval = i
        out = []
        for k in range(len(c)):
            st = c.statuses(k)
            down = int((st == N.EDGE_DOWN).sum())
            cls = {"size": int(c.length[k]), "down": down, "up": int(len(st)) - down, "voters": int(c.voters[k])}
            out.append(dict(cls, representative=int(self.tags[self.ring0[c.representative[k]]])))
            fp = (int(c.hash[k]), int(c.hash2[k]), int(c.length[k]))
            if fp in self.census:
                self.census[fp]["voters"] += cls["voters"]
            else:
                self.census[fp] = dict(cls, ids=frozenset(c.entries(k).tolist()))
        return out

    def _config_census(self, cut, i):
        """the configuration's classes against the decided cut (device ids) -> (census, agreement).  The deciding interval's
        classes are measured by a census with cut= on the device, those of earlier intervals from their lists."""
        cut_set = frozenset(int(x) for x in cut)
        dist = {}
        if self._census_interval == i:
            d = self.cl.proposalCensus(cut=cut)
            for k in range(len(d)):
                dist[(int(d.hash[k]), int(d.hash2[k]), int(d.length[k]))] = (int(d.missing[k]), int(d.extra[k]))
        out = []
        for fp, c in self.census.items():
            missing, extra = dist.get(fp, (len(cut_set - c["ids"]), len(c["ids"] - cut_set)))
            out.append({"size": c["size"], "down": c["down"], "up": c["up"], "voters": c["voters"], "decided": c["ids"] == cut_set,
                        "missing": missing, "extra": extra})
        total = sum(c["voters"] for c in out)
        agreement = sum(c["voters"] for c in out if c["decided"]) / total if total else None
        return out, agreement

    def _announced_flags(self):
        if self._ann is None:
            self._ann = self.cl.readAnnounced()
        return self._ann

    def _overlay(self):
        """(ratio, residual) of the current view's monitoring overlay; (None, None) below 3 members"""
        if self.view.n < 3:
            return None, None
        sp = self.view.overlaySpectrum()
        return sp.ratio, sp.residual

    def _view_change(self, path, value, i):
        t0 = time.perf_counter()
        r = self._proposer if path == "classic" else self.acc.findValue(value)
        assert r >= 0, "a decided value is some acceptor's vote"
        cut = self.cl.getProposal(r)
        census = self._config_census(cut, i) if self.proposal_census else None
        old_tags = np.concatenate([self.tags, np.zeros(self.view.numJoiners(), np.int64)])
        for t, j in self.joiner_id.items():
            old_tags[j] = t
        cut_tags = sorted(int(old_tags[c]) for c in cut)
        mapping = self.view.applyCut(cut)
        new_tags = np.zeros(self.view.n, np.int64)
        kept = mapping >= 0
        new_tags[mapping[kept]] = old_tags[kept]
        self.tags = new_tags
        admitted = set(cut_tags) & set(self.joiners)
        self.flags[list(admitted)] = 0
        self.pending = [t for t in self.pending if t not in admitted]
        before, size_before = self.cfg, self.N
        self.cfg = self.view.currentConfigurationId()
        self._cfg_t["view_change_ms"] += (time.perf_counter() - t0) * 1e3
        t1 = time.perf_counter()
        self.fd.reset()
        self.cl.close()
        self.acc.close()
        times, announced, votes, distinct = self._cfg_t, self.announced, self.votes, len(self.proposal_fps)
        self._new_handles()
        self._register(self.pending)
        times["handles_ms"] += (time.perf_counter() - t1) * 1e3
        self.history.append({"cfg_before": before, "cfg_after": self.cfg, "size_before": size_before, "size": self.view.n,
                             "cut": cut_tags, "path": path, "intervals": i + 1, "announced": announced,
                             "votes": votes, "members": sorted(self.tags.tolist()), "distinct_proposals": distinct, **times})
        if self.overlay_quality:
            self.history[-1]["overlay_ratio"], self.history[-1]["overlay_residual"] = self._overlay()
        if census is not None:
            self.history[-1]["census"], self.history[-1]["agreement"] = census

    # ---- whole runs --------------------------------------------------------------------------------------------------------------
    def run(self, max_intervals):
        """intervals until no flagged node is a member and no joiner is pending (converged), a classic round fails, or
        max_intervals pass without a view change (stalled) -> {"converged", "stalled", "intervals", "stuck"}; stuck = the
        flagged members and pending joiners the run waits on"""
        since, total = 0, 0
        t0 = time.perf_counter()
        while not self.converged():
            if since >= max_intervals:
                break
            rec = self.interval()
            total += 1
            since = 0 if rec["event"].startswith("decided") else since + 1
            if rec["event"] == "stalled":
                break
        done = self.converged()
        stuck = sorted(set(int(t) for t in self.tags[self.flags[self.tags] != 0]) | set(self.pending) | set(self.leaving))
        return {"converged": done, "stalled": not done, "intervals": total, "stuck": stuck,
                "wall_ms": (time.perf_counter() - t0) * 1e3}

    def close(self):
        for h in (self.cl, self.acc, self.fp, self.fd):
            h.close()
