"""Host-side mirror of the fast round of com.vrg.rapid.FastPaxos (FastPaxos.java:125-156): the vote tally of one
configuration, computed by librapid_b200.so on the GPU."""
import ctypes as C

import numpy as np

from . import _native as N


def quorum(membership_size):
    """N - floor((N-1)/4)   (FastPaxos.java:145)"""
    out = C.c_int64(0)
    N.check(N.lib().rapid_fp_quorum(int(membership_size), C.byref(out)))
    return out.value


class TallyResult:
    __slots__ = ("decided", "hash", "hash2", "length", "count", "votes_received", "decided_in")

    def __init__(self, decided, h1, h2, ln, count, received, decided_in=None):
        self.decided, self.hash, self.hash2, self.length, self.count, self.votes_received = decided, h1, h2, ln, count, received
        self.decided_in = decided_in          # index of the tally call that decided (asynchronous tallies only)

    def __repr__(self):
        return "TallyResult(decided=%s, hash=%#x, len=%d, count=%d, votes_received=%d)" % (
            self.decided, self.hash, self.length, self.count, self.votes_received)


class NcclComm:
    """One NCCL communicator per process/GPU for the sharded tally (created from a unique id that rank 0 makes)."""

    @staticmethod
    def unique_id():
        buf = np.zeros(128, np.uint8)
        N.check(N.lib().rapid_comm_unique_id(N.ptr(buf)))
        return buf

    def __init__(self, rank, world, unique_id, device):
        self._h = C.c_void_p()
        uid = N.as_u8(unique_id)
        N.check(N.lib().rapid_comm_init(C.byref(self._h), rank, world, N.ptr(uid), device))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_comm_destroy(self._h)
            self._h = C.c_void_p()


class FastPaxos:
    """FastPaxos(myAddr, configurationId, membershipSize, ...) — fast round only (FastPaxos.java:61-85, :125-156)."""

    def __init__(self, configuration_id, membership_size, sender_capacity=None, device=0):
        self.N = int(membership_size)
        self.cfg = int(configuration_id)
        cap = int(sender_capacity if sender_capacity is not None else membership_size)
        self._h = C.c_void_p()
        N.check(N.lib().rapid_fp_create(C.byref(self._h), self.cfg, self.N, cap, device))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_fp_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _outs():
        return C.c_int32(0), C.c_uint64(0), C.c_uint64(0), C.c_int32(0), C.c_int32(0), C.c_int32(0)

    def handleFastRoundProposals(self, senders, proposal_hash, proposal_hash2=None, proposal_len=None, vote_cfg=None):
        """Apply FastRoundPhase2bMessages in order (handleFastRoundProposal per vote)."""
        s = N.as_i32(senders)
        h1 = np.ascontiguousarray(proposal_hash, np.uint64)
        h2 = None if proposal_hash2 is None else np.ascontiguousarray(proposal_hash2, np.uint64)
        ln = None if proposal_len is None else N.as_i32(proposal_len)
        vc = None if vote_cfg is None else N.as_i64(vote_cfg)
        d, a, b, l, c, r = self._outs()
        N.check(N.lib().rapid_fp_tally(self._h, len(s), N.ptr(s), N.ptr(vc), N.ptr(h1), N.ptr(h2), N.ptr(ln), C.byref(d),
                                       C.byref(a), C.byref(b), C.byref(l), C.byref(c), C.byref(r)))
        return TallyResult(bool(d.value), a.value, b.value, l.value, c.value, r.value)

    def handleFastRoundProposalsFromWire(self, decoder):
        """handleFastRoundProposals over the FastRoundPhase2bMessages of decoder's last decode, on the device.  Votes of another
        configuration are dropped first; one of this configuration from an endpoint outside the dictionary raises
        RapidError(EINVAL) with nothing changed"""
        d, a, b, l, c, r = self._outs()
        N.check(N.lib().rapid_fp_tally_wire(self._h, decoder._h, C.byref(d), C.byref(a), C.byref(b), C.byref(l), C.byref(c), C.byref(r)))
        return TallyResult(bool(d.value), a.value, b.value, l.value, c.value, r.value)

    def tallyCluster(self, cluster, comm=None):
        """Every receiver of `cluster` that announced in the last batch votes for its proposal."""
        d, a, b, l, c, r = self._outs()
        N.check(N.lib().rapid_fp_tally_cd(self._h, cluster._h, comm._h if comm is not None else None, C.byref(d),
                                          C.byref(a), C.byref(b), C.byref(l), C.byref(c), C.byref(r)))
        return TallyResult(bool(d.value), a.value, b.value, l.value, c.value, r.value)

    def tallyClusterAsync(self, cluster, comm=None):
        """enqueue only; result() collects the outcome of the last enqueued tally"""
        N.check(N.lib().rapid_fp_tally_cd_async(self._h, cluster._h, comm._h if comm is not None else None))

    def epochAsync(self, cluster, configuration_id, n_cells, dst_dev, ring_dev, status_dev, comm=None, blocked_dev=0, perm_seed=None):
        """clear() + a new FastPaxos instance + one device-resident alert batch + its tally, enqueued in one call"""
        from . import _native as Nn
        d = None
        if blocked_dev or perm_seed is not None:
            d = Nn.Delivery()
            d.flags = 0
            if blocked_dev:
                d.flags |= Nn.DELIVERY_BLOCKED
                d.blocked = blocked_dev
            if perm_seed is not None:
                d.flags |= Nn.DELIVERY_PERMUTED
                d.perm_seed = perm_seed & 0xFFFFFFFFFFFFFFFF
        self.cfg = int(configuration_id)
        N.check(N.lib().rapid_fp_epoch_async(self._h, cluster._h, comm._h if comm is not None else None, self.cfg, self.N, int(n_cells),
                                             dst_dev, ring_dev, status_dev, None, C.byref(d) if d is not None else None))

    def result(self):
        d, a, b, l, c, r = self._outs()
        k = C.c_int32(-1)
        N.check(N.lib().rapid_fp_result(self._h, C.byref(d), C.byref(a), C.byref(b), C.byref(l), C.byref(c), C.byref(r), C.byref(k)))
        return TallyResult(bool(d.value), a.value, b.value, l.value, c.value, r.value, k.value)

    def reset(self, configuration_id, membership_size=None):
        """the new FastPaxos instance of the next configuration (MembershipService.java:427-429)"""
        self.cfg = int(configuration_id)
        if membership_size is not None:
            self.N = int(membership_size)
        N.check(N.lib().rapid_fp_reset(self._h, self.cfg, self.N))

    def timerStop(self, cluster):
        """milliseconds on the device since cluster.timerStart(), after everything enqueued so far on both handles"""
        a = C.c_float(0)
        N.check(N.lib().rapid_fp_timer_stop(self._h, cluster._h, C.byref(a)))
        return a.value

    def lastLaunches(self):
        a = C.c_int32(0)
        N.check(N.lib().rapid_fp_last_launches(self._h, C.byref(a)))
        return a.value

    def lastDeviceMs(self):
        a = C.c_float(0)
        N.check(N.lib().rapid_fp_last_device_ms(self._h, C.byref(a)))
        return a.value
