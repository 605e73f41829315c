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


class ProposalCensus:
    """The distinct proposals announced in a VirtualCluster's last call (rapid_cd_proposal_census).

    Class i is the i-th distinct (hash, hash2, length) in order of its lowest announcing receiver (representative[i]); voters[i]
    receivers announced it.  entries(i) is its list in canonical ring-0 order (getProposal(representative[i])), statuses(i) the
    NodeStatusChange status of each entry (DOWN: a member, UP: a registered joiner) as VIEW_CHANGE_PROPOSAL hands them out.
    With a cut: in_cut[i] entries of the class are in it, missing[i] = |cut| - in_cut[i], extra[i] = length[i] - in_cut[i];
    without one the three read -1.  classes() is the class of every receiver (-1: did not announce), classes_dev the same array
    in device memory (valid until the next census of the cluster)."""

    def __init__(self, cluster, n_classes, n_entries, cut_len):
        nc, ne = int(n_classes), int(n_entries)
        self._cluster = cluster
        self.hash, self.hash2 = np.zeros(nc, np.uint64), np.zeros(nc, np.uint64)
        self.length, self.voters, self.representative = (np.zeros(nc, np.int32) for _ in range(3))
        self.in_cut = np.zeros(nc, np.int32)
        self.list_off = np.zeros(nc + 1, np.int64)
        self.ids, self.status = np.zeros(ne, np.int32), np.zeros(ne, np.uint8)
        N.check(N.lib().rapid_cd_read_census(cluster._h, N.ptr(self.hash), N.ptr(self.hash2), N.ptr(self.length), N.ptr(self.voters),
                                             N.ptr(self.representative), N.ptr(self.in_cut), N.ptr(self.list_off), N.ptr(self.ids),
                                             N.ptr(self.status)))
        if cut_len is None:
            self.missing = np.full(nc, -1, np.int32)
            self.extra = np.full(nc, -1, np.int32)
        else:
            self.missing = (cut_len - self.in_cut).astype(np.int32)
            self.extra = (self.length - self.in_cut).astype(np.int32)
        p = C.c_void_p()
        N.check(N.lib().rapid_cd_census_classes_dev(cluster._h, C.byref(p)))
        self.classes_dev = p.value or 0

    def __len__(self):
        return len(self.hash)

    def entries(self, i):
        return self.ids[self.list_off[i]: self.list_off[i + 1]]

    def statuses(self, i):
        return self.status[self.list_off[i]: self.list_off[i + 1]]

    def classes(self):
        out = np.zeros(self._cluster.R, np.int32)
        N.check(N.lib().rapid_cd_read_census_classes(self._cluster._h, N.ptr(out)))
        return out


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

    def proposalCensus(self, cut=None):
        """The distinct proposals announced in the last call, counted and listed on the device -> ProposalCensus.  cut: node
        ids to measure each proposal against (missing / extra), e.g. the decided cut."""
        c = None if cut is None else N.as_i32(cut)
        n = 0 if c is None else len(c)
        buf = None if c is None else (c if n else np.zeros(1, np.int32))    # an empty cut is a cut: a non-NULL pointer
        nc, ne = C.c_int64(0), C.c_int64(0)
        N.check(N.lib().rapid_cd_proposal_census(self._h, N.ptr(buf), n, C.byref(nc), C.byref(ne)))
        return ProposalCensus(self, nc.value, ne.value, None if c is None else n)

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
