"""Host-side mirror of com.vrg.rapid.MembershipView over the device-resident K-ring view.

Method names and error behaviour follow rapid/src/main/java/com/vrg/rapid/MembershipView.java so that the parity
tests read like the reference's MembershipViewTest; node ids (ints) stand for Endpoint objects.
All results come from librapid_b200.so (CUDA); nothing is computed here.
"""
import collections
import ctypes as C

import numpy as np

from . import _native as N


OverlaySpectrum = collections.namedtuple("OverlaySpectrum", "lambda2 lambda_min residual steps device_ms lambda_ ratio")


class MembershipView:
    """MembershipView(K, nodeIds, endpoints) bulk constructor (MembershipView.java:74-89).

    hostnames: list of str/bytes (Endpoint.hostname), ports: list of int (Endpoint.port).
    Members get ids 0..n-1 in the given order.
    """

    def __init__(self, K, hostnames=(), ports=(), device=0, _packed=None):
        self.K = int(K)
        self.device = device
        if _packed is not None:
            hb, off, port = _packed
        else:
            hb, off = N.pack_hostnames(hostnames)
            port = N.as_i32(ports)
        n = len(port)
        self.n = n
        self._h = C.c_void_p()
        N.check(N.lib().rapid_view_create(C.byref(self._h), self.K, n, N.ptr(hb), N.ptr(off), N.ptr(port), device))

    @classmethod
    def from_packed(cls, K, host_bytes, host_off, ports, device=0):
        return cls(K, device=device, _packed=(N.as_u8(host_bytes), N.as_i32(host_off), N.as_i32(ports)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_view_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- queries -------------------------------------------------------------------------------
    def getMembershipSize(self):                                   # :425-432
        out = C.c_int64(0)
        N.check(N.lib().rapid_view_size(self._h, C.byref(out)))
        return out.value

    def getRing(self, k):                                          # :380-388
        out = np.empty(max(self.n, 1), np.int32)
        N.check(N.lib().rapid_view_ring(self._h, k, N.ptr(out)))
        return out[: self.n]

    def keys(self, k):
        tot = self.n + self.numJoiners()
        out = np.empty(max(tot, 1), np.int64)
        N.check(N.lib().rapid_view_keys(self._h, k, N.ptr(out)))
        return out[:tot]

    def _row(self, fn, node):
        out = np.empty(self.K, np.int32)
        cnt = C.c_int32(0)
        N.check(fn(self._h, int(node), N.ptr(out), C.byref(cnt)))
        return out[: cnt.value].tolist()

    def getObserversOf(self, node):                                # :210-257
        return self._row(N.lib().rapid_view_observers, node)

    def getSubjectsOf(self, node):                                 # :267-282
        return self._row(N.lib().rapid_view_subjects, node)

    def getExpectedObserversOf(self, hostname, port):              # :292-303
        hb = hostname.encode("utf-8") if isinstance(hostname, str) else bytes(hostname)
        buf = np.frombuffer(hb, dtype=np.uint8).copy() if hb else np.zeros(1, np.uint8)
        out = np.empty(self.K, np.int32)
        cnt = C.c_int32(0)
        N.check(N.lib().rapid_view_expected_observers(self._h, N.ptr(buf), len(hb), int(port), N.ptr(out), C.byref(cnt)))
        return out[: cnt.value].tolist()

    def getRingNumbers(self, observer, subject):                   # :397-418
        m = C.c_uint16(0)
        N.check(N.lib().rapid_view_ring_numbers(self._h, int(observer), int(subject), C.byref(m)))
        return [k for k in range(self.K) if (m.value >> k) & 1]

    def isHostPresent(self, node):                                 # :330-337
        return 0 <= node < self.n

    def tables(self):
        """(observers[n][K], subjects[n][K]) of every member."""
        obs = np.empty((max(self.n, 1), self.K), np.int32)
        subj = np.empty((max(self.n, 1), self.K), np.int32)
        N.check(N.lib().rapid_view_tables(self._h, N.ptr(obs), N.ptr(subj)))
        return obs[: self.n], subj[: self.n]

    def getCurrentConfigurationId(self, id_high, id_low):          # :360-372, :544-556
        hi, lo = N.as_i64(id_high), N.as_i64(id_low)
        out = C.c_int64(0)
        N.check(N.lib().rapid_view_config_id(self._h, N.ptr(hi), N.ptr(lo), len(hi), C.byref(out)))
        return out.value

    def setNodeIds(self, id_high, id_low):
        """NodeIds of the current members (index = node id): identifiersSeen on the device (MembershipView.java:58-60)."""
        hi, lo = N.as_i64(id_high), N.as_i64(id_low)
        assert len(hi) == self.n and len(lo) == self.n
        N.check(N.lib().rapid_view_set_node_ids(self._h, N.ptr(hi), N.ptr(lo)))

    def setJoinerIds(self, first_joiner_id, id_high, id_low):
        hi, lo = N.as_i64(id_high), N.as_i64(id_low)
        N.check(N.lib().rapid_view_set_joiner_ids(self._h, int(first_joiner_id), len(hi), N.ptr(hi), N.ptr(lo)))

    def currentConfigurationId(self):                              # :360-372 from the device-resident identifiersSeen
        out = C.c_int64(0)
        N.check(N.lib().rapid_view_current_config_id(self._h, C.byref(out)))
        return out.value

    def registerJoiners(self, hostnames, ports):
        """ids for endpoints that UP alerts will name (the edgeDst of a join)."""
        hb, off = N.pack_hostnames(hostnames)
        port = N.as_i32(ports)
        first = C.c_int32(0)
        N.check(N.lib().rapid_view_register_joiners(self._h, len(port), N.ptr(hb), N.ptr(off), N.ptr(port), C.byref(first)))
        return list(range(first.value, first.value + len(port)))

    def applyCut(self, cut_ids, want_map=True):
        """decideViewChange (MembershipService.java:385-444): members in the cut leave, registered joiners in it are added;
        the K rings are updated on the device (compaction + sorted merge).  Returns old id -> new id (-1 = gone); detector handles
        on the old view are stale.  Raises UUIDAlreadySeenException (view unchanged) if NodeIds are set and a joiner's was seen."""
        ids = N.as_i32(cut_ids)
        tot = self.n + self.numJoiners()
        mapping = np.empty(max(tot, 1), np.int32) if want_map else None
        N.check(N.lib().rapid_view_apply_cut(self._h, N.ptr(ids), len(ids), N.ptr(mapping)))
        self.n = self.getMembershipSize()
        return mapping[:tot] if want_map else None

    def joinerTables(self):
        """expected observers [n_joiners][K] of the registered joiners"""
        nj = self.numJoiners()
        out = np.empty((max(nj, 1), self.K), np.int32)
        N.check(N.lib().rapid_view_joiner_tables(self._h, N.ptr(out)))
        return out[:nj]

    def numJoiners(self):
        out = C.c_int64(0)
        N.check(N.lib().rapid_view_num_joiners(self._h, C.byref(out)))
        return out.value

    def overlaySpectrum(self, seed=0, tol=1e-3, max_steps=256):
        """Expansion of the monitoring overlay (rapid_view_overlay_spectrum): lambda2 and lambda_min, the largest and smallest
        eigenvalue of the members' observer graph A = sum_k (P_k + P_k^T) below the trivial 2K; lambda_ = max(|lambda2|,
        |lambda_min|) and ratio = lambda_ / 2K, the Rapid paper's expander figure; residual bounds the error of the two values
        (the call stops at residual <= tol * 2K or after max_steps operator applications, steps says how many it spent)."""
        l2, lmin, res = C.c_double(0), C.c_double(0), C.c_double(0)
        steps, ms = C.c_int32(0), C.c_float(0)
        N.check(N.lib().rapid_view_overlay_spectrum(self._h, int(seed) & 0xFFFFFFFFFFFFFFFF, float(tol), int(max_steps), C.byref(l2),
                                                    C.byref(lmin), C.byref(res), C.byref(steps), C.byref(ms)))
        lam = max(abs(l2.value), abs(lmin.value))
        return OverlaySpectrum(l2.value, lmin.value, res.value, steps.value, ms.value, lam, lam / (2.0 * self.K))
