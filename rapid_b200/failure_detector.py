"""Host-side mirror of alert generation (SURVEY.md §8 f4): the K PingPongFailureDetectors of every virtual node
(PingPongFailureDetector.java:38-121, one per entry of getSubjectsOf(myAddr), MembershipService.java:697-707) and the
AlertMessages their notifiers raise (MembershipService.java:472-495), computed by librapid_b200.so (csrc/fd.cu)."""
import ctypes as C

import numpy as np

from . import _native as N

CRASHED, INGRESS_BLOCKED, EGRESS_BLOCKED, BOOTSTRAPPING = 1, 2, 4, 8
FAILURE_THRESHOLD = 10                 # PingPongFailureDetector.java:41
BOOTSTRAP_COUNT_THRESHOLD = 30         # PingPongFailureDetector.java:45


class EdgeFailureDetectors:
    def __init__(self, view, failure_threshold=FAILURE_THRESHOLD, bootstrap_threshold=BOOTSTRAP_COUNT_THRESHOLD):
        self.view = view
        self._h = C.c_void_p()
        N.check(N.lib().rapid_fdet_create(C.byref(self._h), view._h, int(failure_threshold), int(bootstrap_threshold)))
        self.n_alerts = self.n_cells = 0

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_fdet_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        """new configuration: the detectors are cancelled and re-created (MembershipService.java:433-434)"""
        N.check(N.lib().rapid_fdet_reset(self._h))

    def tick(self, node_flags, cfg_id, edge_fail=None):
        """one failure-detector interval of the whole cluster -> (number of AlertMessages, number of cells) raised"""
        nf = N.as_u8(node_flags)
        ef = None if edge_fail is None else N.as_u8(edge_fail)
        a, c = C.c_int64(0), C.c_int64(0)
        N.check(N.lib().rapid_fdet_tick(self._h, N.ptr(nf), N.ptr(ef), int(cfg_id), C.byref(a), C.byref(c)))
        self.n_alerts, self.n_cells = a.value, c.value
        return a.value, c.value

    def tickDevice(self, node_flags_dev, cfg_id, edge_fail_dev=None):
        """tick() with the flags (and per-detector failures) already in device memory (raw pointers); the flags must stay
        there until joinAlerts() of the same interval"""
        a, c = C.c_int64(0), C.c_int64(0)
        N.check(N.lib().rapid_fdet_tick_dev(self._h, node_flags_dev, edge_fail_dev or None, int(cfg_id), C.byref(a), C.byref(c)))
        self.n_alerts, self.n_cells = a.value, c.value
        return a.value, c.value

    def joinAlerts(self, joiner_ids, cfg_id):
        """join phase 2 (MembershipService.java:232-281) in the last tick's interval: every live expected observer of each listed
        registered joiner raises one UP alert; merged per sender after the detectors' alerts, joiners in list order.
        -> (number of AlertMessages, number of cells) of the merged interval"""
        ids = N.as_i32(joiner_ids)
        a, c = C.c_int64(0), C.c_int64(0)
        N.check(N.lib().rapid_fdet_join_alerts(self._h, N.ptr(ids), len(ids), int(cfg_id), C.byref(a), C.byref(c)))
        self.n_alerts, self.n_cells = a.value, c.value
        return a.value, c.value

    def mergeAlerts(self, joiner_ids, leaver_ids, cfg_id):
        """joinAlerts() and graceful leaves (MembershipService.leave :545-565 -> handleLeaveMessage :372-376) in one merge into the
        last tick's interval: every live observer k of each listed member raises one DOWN alert with the ring numbers of that edge,
        repeats kept (K alerts for a leaver whose observers all live).  Per sender: the detectors' alerts, then the join alerts,
        then the leave alerts, each in list order.  One merge per tick.  -> (number of AlertMessages, number of cells)"""
        jids, lids = N.as_i32(joiner_ids), N.as_i32(leaver_ids)
        a, c = C.c_int64(0), C.c_int64(0)
        N.check(N.lib().rapid_fdet_merge_alerts(self._h, N.ptr(jids), len(jids), N.ptr(lids), len(lids), int(cfg_id), C.byref(a),
                                                C.byref(c)))
        self.n_alerts, self.n_cells = a.value, c.value
        return a.value, c.value

    def alerts(self):
        """[(observer, subject, [ring numbers])] of the last tick, in the order the notifiers fired"""
        n = self.n_alerts
        o, s, m = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint16)
        N.check(N.lib().rapid_fdet_read_alerts(self._h, N.ptr(o), N.ptr(s), N.ptr(m)))
        return [(int(o[i]), int(s[i]), [r for r in range(16) if (int(m[i]) >> r) & 1]) for i in range(n)]

    def cells(self):
        """(src, dst, ring, status, cfg) of the interval's cells"""
        n = self.n_cells
        src, dst = np.zeros(n, np.int32), np.zeros(n, np.int32)
        ring, status, cfg = np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.int64)
        N.check(N.lib().rapid_fdet_read_cells(self._h, N.ptr(src), N.ptr(dst), N.ptr(ring), N.ptr(status), N.ptr(cfg)))
        return src, dst, ring, status, cfg

    def senderBatches(self):
        """batch offsets of the last tick's cells grouped per sender, the way AlertBatcher ships them (one BatchedAlertMessage
        per observer and window, MembershipService.java:613-637): feed VirtualCluster.handleBatchesDevice"""
        cap = self.n_cells + 2
        off = np.zeros(cap, np.int64)
        nb = C.c_int64(0)
        N.check(N.lib().rapid_fdet_sender_batches(self._h, N.ptr(off), cap, C.byref(nb)))
        return off[: nb.value + 1]

    def cellsDevice(self):
        p = [C.c_void_p() for _ in range(5)]
        N.check(N.lib().rapid_fdet_cells_dev(self._h, *[C.byref(x) for x in p]))
        return tuple(x.value for x in p)

    def state(self, node, k):
        """(failureCount, notified) of node's k-th detector"""
        a, b = C.c_int32(0), C.c_int32(0)
        N.check(N.lib().rapid_fdet_state(self._h, int(node), int(k), C.byref(a), C.byref(b)))
        return a.value, bool(b.value)

    def lastDeviceMs(self):
        out = C.c_float(0)
        N.check(N.lib().rapid_fdet_last_device_ms(self._h, C.byref(out)))
        return out.value
