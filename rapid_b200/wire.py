"""Wire-format ingest (SURVEY.md §8 f3): serialized rapid.proto messages -> alert cells / votes, decoded on the GPU by
librapid_b200.so (csrc/wire.cu), consensus messages included.  This is the step the reference's gRPC server does before
MembershipService.handleMessage(RapidRequest) (MembershipService.java:174): no Python protobuf runtime is involved."""
import ctypes as C

import numpy as np

from . import _native as N


class DecodedAlerts:
    __slots__ = ("n_messages", "n_cells", "n_dropped", "n_new_joiners", "sender")

    def __init__(self, n_messages, n_cells, n_dropped, n_new_joiners, sender):
        self.n_messages, self.n_cells, self.n_dropped, self.n_new_joiners, self.sender = n_messages, n_cells, n_dropped, n_new_joiners, sender

    def __repr__(self):
        return "DecodedAlerts(messages=%d, cells=%d, dropped=%d, new_joiners=%d, sender=%d)" % (
            self.n_messages, self.n_cells, self.n_dropped, self.n_new_joiners, self.sender)


class EncodedMessages:
    """The outputs of one encode, copied to the host: message i = headers[header_off[i]:header_off[i+1]] ++ body body_ids[i]
    (none when -1).  Messages that carry the same list share one body."""

    def __init__(self, headers, header_off, body_ids, bodies, body_off, sizes, senders):
        self.headers, self.header_off, self.body_ids, self.bodies, self.body_off = headers, header_off, body_ids, bodies, body_off
        self._sizes = sizes
        self.senders = senders                 # view id of each message's sender

    def __len__(self):
        return len(self.body_ids)

    def header(self, i):
        return self.headers[self.header_off[i]:self.header_off[i + 1]].tobytes()

    def body(self, b):
        return self.bodies[self.body_off[b]:self.body_off[b + 1]].tobytes()

    def message(self, i):
        b = int(self.body_ids[i])
        return self.header(i) + (self.body(b) if b >= 0 else b"")

    def sizes(self):
        """bytes of every message, header + body, as the device computed them"""
        return self._sizes

    def __repr__(self):
        return "EncodedMessages(messages=%d, bodies=%d, bytes=%d)" % (len(self), len(self.body_off) - 1, int(self._sizes.sum()))


class WireDecoder:
    """Owns the Endpoint{hostname, port} -> id table of a MembershipView on the device."""

    def __init__(self, view):
        self.view = view
        self._h = C.c_void_p()
        N.check(N.lib().rapid_wire_create(C.byref(self._h), view._h))
        self._last = None
        self._n_cons = 0                     # messages of the last consensus decode

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_wire_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def setConfiguration(self, cfg_id):
        """only UP alerts of this configuration may register joiners from now on (MembershipService.java:653)"""
        N.check(N.lib().rapid_wire_set_configuration(self._h, int(cfg_id)))

    def decodeBatchedAlertMessage(self, data, is_request=False):
        """bytes of a BatchedAlertMessage (or of the RapidRequest carrying it) -> DecodedAlerts; the cells stay on the device"""
        buf = np.frombuffer(bytes(data), dtype=np.uint8) if len(data) else np.zeros(1, np.uint8)
        m, c, d, j, s = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int32(-1)
        self._n_cons = 0
        N.check(N.lib().rapid_wire_decode_alerts(self._h, N.ptr(buf), len(data), N.WIRE_REQUEST if is_request else 0, C.byref(m),
                                                 C.byref(c), C.byref(d), C.byref(j), C.byref(s)))
        self._last = DecodedAlerts(m.value, c.value, d.value, j.value, s.value)
        return self._last

    def cells(self):
        """host copies of the last decode: (src, dst, ring, status, cfg)"""
        n = self._last.n_cells if self._last else 0
        src, dst = np.zeros(n, np.int32), np.zeros(n, np.int32)
        ring, status, cfg = np.zeros(n, np.uint8), np.zeros(n, np.uint8), np.zeros(n, np.int64)
        N.check(N.lib().rapid_wire_read_cells(self._h, N.ptr(src), N.ptr(dst), N.ptr(ring), N.ptr(status), N.ptr(cfg)))
        return src, dst, ring, status, cfg

    def cellsDevice(self):
        """device pointers (src, dst, ring, status, cfg) of the last decode, for rapid_cd_apply_batch_dev"""
        p = [C.c_void_p() for _ in range(5)]
        N.check(N.lib().rapid_wire_cells_dev(self._h, *[C.byref(x) for x in p]))
        return tuple(x.value for x in p)

    def messages(self):
        """per AlertMessage of the last decode: dict of arrays dst, status, n_rings, node_high, node_low, has_node_id,
        meta_off, meta_len"""
        n = self._last.n_messages if self._last else 0
        out = {"dst": np.zeros(n, np.int32), "status": np.zeros(n, np.uint8), "n_rings": np.zeros(n, np.int32),
               "node_high": np.zeros(n, np.int64), "node_low": np.zeros(n, np.int64), "has_node_id": np.zeros(n, np.uint8),
               "meta_off": np.zeros(n, np.int64), "meta_len": np.zeros(n, np.int32)}
        N.check(N.lib().rapid_wire_read_messages(self._h, *[N.ptr(out[k]) for k in ("dst", "status", "n_rings", "node_high", "node_low",
                                                                                   "has_node_id", "meta_off", "meta_len")]))
        return out

    @staticmethod
    def _pack(messages):
        n = len(messages)
        off = np.zeros(n + 1, np.int64)
        if n:
            off[1:] = np.cumsum([len(m) for m in messages])
        joined = b"".join(bytes(m) for m in messages)
        return n, off, np.frombuffer(joined, dtype=np.uint8) if joined else np.zeros(1, np.uint8)

    def decodeFastRoundPhase2bMessages(self, messages, is_request=False):
        """list of serialized FastRoundPhase2bMessages -> (sender, cfg, hash, hash2, len) arrays"""
        n, off, buf = self._pack(messages)
        self._n_cons = 0
        s, c = np.zeros(n, np.int32), np.zeros(n, np.int64)
        h1, h2, ln = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.int32)
        N.check(N.lib().rapid_wire_decode_votes(self._h, N.ptr(buf), N.ptr(off), n, N.WIRE_REQUEST if is_request else 0, N.ptr(s),
                                                N.ptr(c), N.ptr(h1), N.ptr(h2), N.ptr(ln)))
        self._n_cons = n
        return s, c, h1, h2, ln

    def decodeConsensusMessages(self, kind, messages, is_request=False):
        """serialized consensus messages of one kind (N.WIRE_FAST_ROUND_PHASE2B, N.WIRE_PHASE1A, N.WIRE_PHASE1B,
        N.WIRE_PHASE2A, N.WIRE_PHASE2B) decoded on the device, where Paxos.handlePhase1bFromWire / handlePhase2bFromWire and
        FastPaxos.handleFastRoundProposalsFromWire take them.  -> (messages whose sender is unknown, unknown list entries)"""
        n, off, buf = self._pack(messages)
        self._n_cons = 0
        a, b = C.c_int64(0), C.c_int64(0)
        N.check(N.lib().rapid_wire_decode_consensus(self._h, int(kind), N.ptr(buf), N.ptr(off), n, N.WIRE_REQUEST if is_request else 0,
                                                    C.byref(a), C.byref(b)))
        self._n_cons = n
        return a.value, b.value

    def consensusMessages(self):
        """per message of the last consensus decode: dict of arrays sender, cfg, rnd_round, rnd_node, vrnd_round, vrnd_node,
        hash, hash2, len"""
        n = getattr(self, "_n_cons", 0)
        out = {"sender": np.zeros(n, np.int32), "cfg": np.zeros(n, np.int64), "rnd_round": np.zeros(n, np.int32),
               "rnd_node": np.zeros(n, np.int32), "vrnd_round": np.zeros(n, np.int32), "vrnd_node": np.zeros(n, np.int32),
               "hash": np.zeros(n, np.uint64), "hash2": np.zeros(n, np.uint64), "len": np.zeros(n, np.int32)}
        N.check(N.lib().rapid_wire_read_consensus(self._h, *[N.ptr(out[k]) for k in ("sender", "cfg", "rnd_round", "rnd_node", "vrnd_round",
                                                                                   "vrnd_node", "hash", "hash2", "len")]))
        return out

    def consensusValue(self, index):
        """the list of message `index` of the last consensus decode as ids in wire order (-1: endpoint not in the dictionary)"""
        ln = C.c_int32(0)
        N.check(N.lib().rapid_wire_consensus_value(self._h, int(index), None, 0, C.byref(ln)))
        ids = np.zeros(max(ln.value, 1), np.int32)
        N.check(N.lib().rapid_wire_consensus_value(self._h, int(index), N.ptr(ids), ln.value, C.byref(ln)))
        return ids[:ln.value].tolist()

    def lastDeviceMs(self):
        out = C.c_float(0)
        N.check(N.lib().rapid_wire_last_device_ms(self._h, C.byref(out)))
        return out.value

    # ---- egress: the messages the virtual nodes send, encoded on the device (csrc/wire_encode.cu) ----
    def encodeAlertBatches(self, detectors, as_request=False):
        """one BatchedAlertMessage per sender of the last interval of an EdgeFailureDetectors -> EncodedMessages"""
        N.check(N.lib().rapid_wire_encode_alert_batches(self._h, detectors._h, N.WIRE_REQUEST if as_request else 0, None, None))
        return self.encoded()

    def encodeVotes(self, detector, cfg_id, as_request=False):
        """one FastRoundPhase2bMessage per receiver of a MembershipServiceCutDetector that announced in its last call"""
        N.check(N.lib().rapid_wire_encode_votes(self._h, detector._h, int(cfg_id), N.WIRE_REQUEST if as_request else 0, None, None))
        return self.encoded()

    def encodePhase1b(self, acceptors, detector=None, as_request=False):
        """one Phase1bMessage per answer of a PaxosAcceptors' last handlePhase1aMessage; vval lists from the votes this handle
        encoded, else from the detector whose receivers are the acceptors"""
        N.check(N.lib().rapid_wire_encode_phase1b(self._h, acceptors._h, detector._h if detector is not None else None,
                                                  N.WIRE_REQUEST if as_request else 0, None, None))
        return self.encoded()

    def encodePhase2b(self, acceptors, detector=None, as_request=False):
        """one Phase2bMessage per answer of a PaxosAcceptors' last handlePhase2aMessage"""
        N.check(N.lib().rapid_wire_encode_phase2b(self._h, acceptors._h, detector._h if detector is not None else None,
                                                  N.WIRE_REQUEST if as_request else 0, None, None))
        return self.encoded()

    def encodedSenders(self):
        """view id of the sender of every message of the last encode"""
        n = self.encodedCounts()[0]
        out = np.zeros(n, np.int32)
        N.check(N.lib().rapid_wire_read_encoded_senders(self._h, N.ptr(out) if n else None))
        return out

    def encodedCounts(self):
        """(messages, header bytes, bodies, body bytes) of the last encode"""
        v = [C.c_int64(0) for _ in range(4)]
        N.check(N.lib().rapid_wire_encoded_counts(self._h, *[C.byref(x) for x in v]))
        return tuple(x.value for x in v)

    def encodedSizes(self):
        """bytes of every message of the last encode, header + body, computed on the device"""
        n = self.encodedCounts()[0]
        out = np.zeros(n, np.int64)
        N.check(N.lib().rapid_wire_read_encoded_sizes(self._h, N.ptr(out) if n else None))
        return out

    def encoded(self):
        """host copies of the last encode -> EncodedMessages"""
        n, hb, nb, bb = self.encodedCounts()
        hdr, hoff, bid = np.zeros(max(hb, 1), np.uint8), np.zeros(n + 1, np.int64), np.zeros(max(n, 1), np.int32)
        bodies, boff = np.zeros(max(bb, 1), np.uint8), np.zeros(nb + 1, np.int64)
        N.check(N.lib().rapid_wire_read_encoded(self._h, N.ptr(hdr), N.ptr(hoff), N.ptr(bid), N.ptr(bodies), N.ptr(boff)))
        return EncodedMessages(hdr[:hb], hoff, bid[:n], bodies[:bb], boff, self.encodedSizes(), self.encodedSenders())
