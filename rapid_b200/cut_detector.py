"""Host-side mirrors of com.vrg.rapid.MultiNodeCutDetector (RAW handles, one or more bare detectors) and of the
MembershipService alert-batch handler for R virtual nodes (SERVICE handles).

Reference: rapid/src/main/java/com/vrg/rapid/MultiNodeCutDetector.java, MembershipService.java:300-354, :644-685.
Everything is computed by librapid_b200.so on the GPU; a missing library / device raises.
"""
import ctypes as C

import numpy as np

from . import _native as N
from .membership_view import MembershipView

UP, DOWN = N.EDGE_UP, N.EDGE_DOWN


def proposal_fingerprint(ids):
    """(h1, h2) of a set of node ids — the identity votes are counted under (rapid_proposal_fingerprint)."""
    a = N.as_i32(ids)
    h1, h2 = C.c_uint64(0), C.c_uint64(0)
    N.check(N.lib().rapid_proposal_fingerprint(N.ptr(a), len(a), C.byref(h1), C.byref(h2)))
    return h1.value, h2.value


class MultiNodeCutDetector:
    """MultiNodeCutDetector(K, H, L) (MultiNodeCutDetector.java:51-60) — K comes from the view.

    n_detectors independent detectors all fed the same calls (tests use 1).  Node ids stand for Endpoints.
    """

    def __init__(self, view: MembershipView, H, L, n_detectors=1):
        self.view = view
        self._h = C.c_void_p()
        rc = N.lib().rapid_cd_create(C.byref(self._h), view._h, int(H), int(L), int(n_detectors), 0, N.CD_RAW, 0)
        if rc == N.EINVAL:
            raise ValueError(N.last_error())          # IllegalArgumentException (:52-55)
        N.check(rc)
        self._cap = 1024

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_cd_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def aggregateForProposal(self, src, dst, status, ring_numbers, detector=0):     # :76-82
        rings = N.as_u8(ring_numbers if hasattr(ring_numbers, "__len__") else [ring_numbers])
        n = len(rings)
        srcs = N.as_i32([src] * n)
        dsts = N.as_i32([dst] * n)
        st = N.as_u8([status] * n)
        out = np.empty(self._cap, np.int32)
        cnt = C.c_int32(0)
        N.check(N.lib().rapid_cd_aggregate(self._h, n, N.ptr(srcs), N.ptr(dsts), N.ptr(rings), N.ptr(st), detector,
                                           N.ptr(out), self._cap, C.byref(cnt)))
        return out[: cnt.value].tolist()

    def invalidateFailingEdges(self, detector=0):                                   # :137-164
        out = np.empty(self._cap, np.int32)
        cnt = C.c_int32(0)
        N.check(N.lib().rapid_cd_invalidate(self._h, detector, N.ptr(out), self._cap, C.byref(cnt)))
        return out[: cnt.value].tolist()

    def getNumProposals(self, detector=0):                                          # :62-66
        out = C.c_int32(0)
        N.check(N.lib().rapid_cd_num_proposals(self._h, detector, C.byref(out)))
        return out.value

    def clear(self):                                                                # :169-178
        N.check(N.lib().rapid_cd_clear(self._h))


class AlertBatchResult:
    __slots__ = ("proposal_hash", "proposal_hash2", "proposal_len", "announced")

    def __init__(self, h1, h2, ln, ann):
        self.proposal_hash, self.proposal_hash2, self.proposal_len, self.announced = h1, h2, ln, ann


class VirtualCluster:
    """The cut detectors + announcedProposal flags of R virtual nodes (MembershipService.java:300-354 for each).

    kernel: "auto" (subject-bucketed kernels), "sweep" (per-cell kernel) or "bucketed".
    Receiver r is the node at ring-0 position receiver_begin + r.
    """

    def __init__(self, view: MembershipView, H, L, n_receivers=None, receiver_begin=0, kernel="auto", max_subjects=0, log=False):
        self.view = view
        self.R = int(view.n if n_receivers is None else n_receivers)
        self.receiver_begin = int(receiver_begin)
        flags = {"auto": N.CD_SERVICE, "sweep": N.CD_SWEEP, "bucketed": N.CD_BUCKETED}[kernel]
        if log:
            flags |= N.CD_LOG              # keep the epoch's cells: getNumProposals on the bucketed kernels
        self._h = C.c_void_p()
        rc = N.lib().rapid_cd_create(C.byref(self._h), view._h, int(H), int(L), self.R, self.receiver_begin, flags,
                                     int(max_subjects))
        if rc == N.EINVAL:
            raise ValueError(N.last_error())
        N.check(rc)
        self._keep = None

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_cd_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _delivery(self, blocked, bitmap, perm_seed, batch_order_seed=None):
        if blocked is None and bitmap is None and perm_seed is None and batch_order_seed is None:
            return None
        d = N.Delivery()
        keep = []
        d.flags = 0
        if blocked is not None:
            b = N.as_u8(blocked)
            assert len(b) == self.R
            keep.append(b)
            d.flags |= N.DELIVERY_BLOCKED
            d.blocked = b.ctypes.data
        if bitmap is not None:
            m = np.ascontiguousarray(bitmap, np.uint32)
            keep.append(m)
            d.flags |= N.DELIVERY_BITMAP
            d.bitmap = m.ctypes.data
        if perm_seed is not None:
            d.flags |= N.DELIVERY_PERMUTED
            d.perm_seed = perm_seed & 0xFFFFFFFFFFFFFFFF
        if batch_order_seed is not None:
            d.flags |= N.DELIVERY_SHUFFLED_BATCHES
            d.perm_seed = batch_order_seed & 0xFFFFFFFFFFFFFFFF
        self._keep = keep
        return d

    def handleBatch(self, cfg_id, src, dst, ring, status, cell_cfg=None, blocked=None, bitmap=None, perm_seed=None,
                    read_outputs=True):
        """One BatchedAlertMessage worth of cells delivered to every receiver."""
        dst = N.as_i32(dst)
        A = len(dst)
        src = N.as_i32(src) if src is not None else np.zeros(max(A, 1), np.int32)
        ring = N.as_u8(ring)
        status = N.as_u8(status)
        cc = None if cell_cfg is None else N.as_i64(cell_cfg)
        d = self._delivery(blocked, bitmap, perm_seed)
        if read_outputs:
            h1 = np.zeros(self.R, np.uint64)
            h2 = np.zeros(self.R, np.uint64)
            ln = np.zeros(self.R, np.int32)
            ann = np.zeros(self.R, np.uint8)
        else:
            h1 = h2 = ln = ann = None
        N.check(N.lib().rapid_cd_apply_batch(self._h, int(cfg_id), A, N.ptr(src), N.ptr(dst), N.ptr(ring), N.ptr(status),
                                             N.ptr(cc), C.byref(d) if d is not None else None, N.ptr(h1), N.ptr(h2),
                                             N.ptr(ln), N.ptr(ann)))
        return AlertBatchResult(h1, h2, ln, ann) if read_outputs else None

    def handleBatchDevice(self, cfg_id, n_cells, dst_dev, ring_dev, status_dev, cell_cfg_dev=0, blocked_dev=0, perm_seed=None,
                          wait=False):
        """Cell arrays already resident in device memory (raw device pointers).  wait=False only ENQUEUES the batch
        (rapid_cd_apply_batch_dev_async): its status is collected by sync() / FastPaxos.tallyCluster."""
        d = None
        if blocked_dev or perm_seed is not None:
            d = N.Delivery()
            d.flags = 0
            if blocked_dev:
                d.flags |= N.DELIVERY_BLOCKED
                d.blocked = blocked_dev
            if perm_seed is not None:
                d.flags |= N.DELIVERY_PERMUTED
                d.perm_seed = perm_seed & 0xFFFFFFFFFFFFFFFF
        fn = N.lib().rapid_cd_apply_batch_dev if wait else N.lib().rapid_cd_apply_batch_dev_async
        N.check(fn(self._h, int(cfg_id), int(n_cells), None, dst_dev, ring_dev, status_dev, cell_cfg_dev or None,
                   C.byref(d) if d is not None else None))

    def timerStart(self):
        N.check(N.lib().rapid_cd_timer_start(self._h))

    def sync(self):
        """wait for asynchronous batches; raises if one of them failed"""
        N.check(N.lib().rapid_cd_sync(self._h))

    def handleBatches(self, cfg_id, src, dst, ring, status, batch_off, cell_cfg=None, blocked=None, bitmap=None, perm_seed=None,
                      read_outputs=True, batch_order_seed=None):
        """A sequence of BatchedAlertMessages (batch b = cells batch_off[b]:batch_off[b+1]) delivered in order, with the
        announcedProposal gating between them (MembershipService.java:318-319).  perm_seed: batch b reaches every receiver in
        its own order, seeded perm_seed + b (bucketed handles).  batch_order_seed: every receiver meets the batches in its own
        order instead, seeded batch_order_seed (RAPID_DELIVERY_SHUFFLED_BATCHES; sweep handles, cells of a batch in array order).
        -> (AlertBatchResult, announced_in): announced_in[r] = index of the batch in which receiver r announced, -1 if none."""
        dst = N.as_i32(dst)
        A = len(dst)
        src = N.as_i32(src) if src is not None else np.zeros(max(A, 1), np.int32)
        ring, status = N.as_u8(ring), N.as_u8(status)
        off = N.as_i64(batch_off)
        cc = None if cell_cfg is None else N.as_i64(cell_cfg)
        d = self._delivery(blocked, bitmap, perm_seed, batch_order_seed)
        if not read_outputs:
            N.check(N.lib().rapid_cd_apply_batches(self._h, int(cfg_id), A, N.ptr(src), N.ptr(dst), N.ptr(ring), N.ptr(status), N.ptr(cc),
                                                   len(off) - 1, N.ptr(off), C.byref(d) if d is not None else None, None, None, None,
                                                   None, None))
            return None, None
        h1, h2 = np.zeros(self.R, np.uint64), np.zeros(self.R, np.uint64)
        ln, ann, ain = np.zeros(self.R, np.int32), np.zeros(self.R, np.uint8), np.zeros(self.R, np.int32)
        N.check(N.lib().rapid_cd_apply_batches(self._h, int(cfg_id), A, N.ptr(src), N.ptr(dst), N.ptr(ring), N.ptr(status), N.ptr(cc),
                                               len(off) - 1, N.ptr(off), C.byref(d) if d is not None else None, N.ptr(h1), N.ptr(h2),
                                               N.ptr(ln), N.ptr(ann), N.ptr(ain)))
        return AlertBatchResult(h1, h2, ln, ann), ain

    def handleBatchesDevice(self, cfg_id, n_cells, dst_dev, ring_dev, status_dev, batch_off, cell_cfg_dev=0, blocked_dev=0, perm_seed=None,
                            batch_order_seed=None):
        """handleBatches with the cell arrays resident in device memory (raw device pointers; batch_off on the host)."""
        d = None
        if blocked_dev or perm_seed is not None or batch_order_seed is not None:
            d = N.Delivery()
            d.flags = 0
            if blocked_dev:
                d.flags |= N.DELIVERY_BLOCKED
                d.blocked = blocked_dev
            if perm_seed is not None:
                d.flags |= N.DELIVERY_PERMUTED
                d.perm_seed = perm_seed & 0xFFFFFFFFFFFFFFFF
            if batch_order_seed is not None:
                d.flags |= N.DELIVERY_SHUFFLED_BATCHES
                d.perm_seed = batch_order_seed & 0xFFFFFFFFFFFFFFFF
        off = N.as_i64(batch_off)
        N.check(N.lib().rapid_cd_apply_batches_dev(self._h, int(cfg_id), int(n_cells), None, dst_dev, ring_dev, status_dev,
                                                   cell_cfg_dev or None, len(off) - 1, N.ptr(off), C.byref(d) if d is not None else None))

    def readAnnouncedIn(self):
        out = np.zeros(self.R, np.int32)
        N.check(N.lib().rapid_cd_read_announced_in(self._h, N.ptr(out)))
        return out

    def sequenceStats(self):
        """(sequences served in one pass, sequences replayed batch by batch)"""
        a, b = C.c_int32(0), C.c_int32(0)
        N.check(N.lib().rapid_cd_sequence_stats(self._h, C.byref(a), C.byref(b), None, None))
        return a.value, b.value

    def sequenceRefusal(self):
        """receivers that failed premise A1 / A2 in the last refused one-pass attempt"""
        a, b = C.c_int32(0), C.c_int32(0)
        N.check(N.lib().rapid_cd_sequence_stats(self._h, None, None, C.byref(a), C.byref(b)))
        return a.value, b.value

    def readOutputs(self):
        h1 = np.zeros(self.R, np.uint64)
        h2 = np.zeros(self.R, np.uint64)
        ln = np.zeros(self.R, np.int32)
        ann = np.zeros(self.R, np.uint8)
        N.check(N.lib().rapid_cd_read_outputs(self._h, N.ptr(h1), N.ptr(h2), N.ptr(ln), N.ptr(ann)))
        return AlertBatchResult(h1, h2, ln, ann)

    def readAnnounced(self):
        """announcedProposal of every receiver (1 B each), without the proposal fingerprints readOutputs() copies too"""
        ann = np.zeros(self.R, np.uint8)
        N.check(N.lib().rapid_cd_read_outputs(self._h, None, None, None, N.ptr(ann)))
        return ann

    def getProposal(self, receiver, cap=1 << 16):
        out = np.empty(cap, np.int32)
        cnt = C.c_int32(0)
        N.check(N.lib().rapid_cd_get_proposal(self._h, int(receiver), N.ptr(out), cap, C.byref(cnt)))
        if cnt.value > cap:
            return self.getProposal(receiver, cnt.value)
        return out[: cnt.value].tolist()

    def getNumProposals(self, receiver):
        out = C.c_int32(0)
        N.check(N.lib().rapid_cd_num_proposals(self._h, int(receiver), C.byref(out)))
        return out.value

    def clear(self):
        N.check(N.lib().rapid_cd_clear(self._h))

    def debugMasks(self, receiver, cap=1 << 16):
        ids = np.empty(cap, np.int32)
        masks = np.empty(cap, np.uint16)
        n = C.c_int32(0)
        N.check(N.lib().rapid_cd_debug_masks(self._h, int(receiver), N.ptr(ids), N.ptr(masks), cap, C.byref(n)))
        if n.value > cap:
            return self.debugMasks(receiver, n.value)
        return dict(zip(ids[: n.value].tolist(), masks[: n.value].tolist()))

    def debugCounters(self, receiver):
        a, b = C.c_int32(0), C.c_int32(0)
        N.check(N.lib().rapid_cd_debug_counters(self._h, int(receiver), C.byref(a), C.byref(b)))
        return a.value, bool(b.value)

    def debugStats(self):
        """(receivers resolved by exact interval analysis, invalidation work-list pairs, batch subjects, valid cells)"""
        a, b, c, d = C.c_int32(0), C.c_int32(0), C.c_int32(0), C.c_int32(0)
        N.check(N.lib().rapid_cd_debug_stats(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)))
        return a.value, b.value, c.value, d.value

    def debugGrid(self):
        """(subject chunks of the last batch's apply kernel, blocks of its k_prepare grid)"""
        a, b = C.c_int32(0), C.c_int32(0)
        N.check(N.lib().rapid_cd_debug_grid(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def lastPath(self):
        a, b = C.c_int32(0), C.c_int32(0)
        N.check(N.lib().rapid_cd_last_path(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def lastDeviceMs(self):
        a, b = C.c_float(0), C.c_float(0)
        N.check(N.lib().rapid_cd_last_device_ms(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value
