"""Host-side mirror of com.vrg.rapid.Paxos (Paxos.java) — the classic-Paxos fallback of the consensus step, computed
by librapid_b200.so on the GPU (csrc/classic_paxos.cu).

Paxos            one node's coordinator + learner tallies (handlePhase1bMessage :159-191, handlePhase2bMessage :223-236,
                 selectProposalUsingCoordinatorRule :271-328), batches of messages in arrival order.
PaxosAcceptors   the acceptor registers (rnd, vrnd, vval) of R virtual nodes (handlePhase1aMessage :120-151,
                 handlePhase2aMessage :198-216, registerFastRoundVote :244-257).  Several of them with disjoint
                 acceptor_begin ranges, on one GPU or on every rank of an NcclComm, feed one Paxos through
                 Paxos.handlePhase1bFromAcceptorShards / handlePhase2bFromAcceptorShards, as one handle over their union would.

A value (List<Endpoint>) is an opaque (hash, hash2, len) triple; len == 0 is the empty list.  A rank is (round, nodeIndex).
"""
import ctypes as C

import numpy as np

from . import _native as N


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _split_ranks(ranks, n):
    r = np.asarray(ranks, dtype=np.int64).reshape(n, 2) if n else np.zeros((0, 2), np.int64)
    return N.as_i32(r[:, 0]), N.as_i32(r[:, 1])


class Phase1bResult:
    __slots__ = ("proposed", "trigger_index", "cval", "n_messages")

    def __init__(self, proposed, trigger_index, cval, n_messages):
        self.proposed, self.trigger_index, self.cval, self.n_messages = proposed, trigger_index, cval, n_messages

    def __repr__(self):
        return "Phase1bResult(proposed=%s, trigger_index=%d, cval=%s, n_messages=%d)" % (
            self.proposed, self.trigger_index, self.cval, self.n_messages)


class Phase2bResult:
    __slots__ = ("decided", "decided_index", "decision")

    def __init__(self, decided, decided_index, decision):
        self.decided, self.decided_index, self.decision = decided, decided_index, decision

    def __repr__(self):
        return "Phase2bResult(decided=%s, decided_index=%d, decision=%s)" % (self.decided, self.decided_index, self.decision)


class Paxos:
    """Paxos(myAddr, configurationId, N, ...) (Paxos.java:76-90): the tallies of one node."""

    def __init__(self, configuration_id, membership_size, message_capacity=None, device=0):
        self.cfg, self.N = int(configuration_id), int(membership_size)
        cap = int(message_capacity if message_capacity is not None else max(2 * self.N, 64))
        self._h = C.c_void_p()
        N.check(N.lib().rapid_px_create(C.byref(self._h), self.cfg, self.N, cap, device))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_px_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, configuration_id, membership_size=None):
        """the Paxos of the next configuration (FastPaxos.java:86) on the same buffers"""
        self.cfg = int(configuration_id)
        self.N = int(self.N if membership_size is None else membership_size)
        N.check(N.lib().rapid_px_reset(self._h, self.cfg, self.N))

    def startPhase1a(self, round_, node_index):
        """:98-113 — node_index stands for myAddr.hashCode().  -> True iff a Phase1aMessage(rank) goes out"""
        out = C.c_int32(0)
        N.check(N.lib().rapid_px_start_phase1a(self._h, int(round_), int(node_index), C.byref(out)))
        return bool(out.value)

    def selectProposalUsingCoordinatorRule(self, vrnd, vval_hash, vval_len, vval_hash2=None):
        """:271-328 — vrnd: (n, 2) ranks.  -> index of the message whose vval is chosen, -1 for the empty list.
        Raises RapidError(EINVAL) on an empty list (the reference throws IllegalArgumentException)."""
        n = len(vval_len)
        r0, r1 = _split_ranks(vrnd, n)
        h1, ln = _u64(vval_hash), N.as_i32(vval_len)
        h2 = None if vval_hash2 is None else _u64(vval_hash2)
        out = C.c_int64(-2)
        N.check(N.lib().rapid_px_coordinator_rule(self._h, n, N.ptr(r0), N.ptr(r1), N.ptr(h1), N.ptr(h2), N.ptr(ln), C.byref(out)))
        return out.value

    @staticmethod
    def _p1_outs():
        return C.c_int32(0), C.c_int64(-1), C.c_uint64(0), C.c_uint64(0), C.c_int32(0), C.c_int64(0)

    @staticmethod
    def _p1_result(o):
        p, t, a, b, l, m = o
        return Phase1bResult(bool(p.value), t.value, (a.value, b.value, l.value) if l.value else None, m.value)

    def handlePhase1bMessages(self, rnd, vrnd, vval_hash, vval_len, vval_hash2=None, msg_cfg=None):
        """:159-191 over a batch in arrival order"""
        n = len(vval_len)
        a0, a1 = _split_ranks(rnd, n)
        b0, b1 = _split_ranks(vrnd, n)
        h1, ln = _u64(vval_hash), N.as_i32(vval_len)
        h2 = None if vval_hash2 is None else _u64(vval_hash2)
        mc = None if msg_cfg is None else N.as_i64(msg_cfg)
        o = self._p1_outs()
        N.check(N.lib().rapid_px_phase1b(self._h, n, N.ptr(mc), N.ptr(a0), N.ptr(a1), N.ptr(b0), N.ptr(b1), N.ptr(h1), N.ptr(h2),
                                         N.ptr(ln), *[C.byref(x) for x in o]))
        return self._p1_result(o)

    def handlePhase1bFromAcceptors(self, acceptors, perm_seed=0):
        """the Phase1b answers of one PaxosAcceptors, read on the device: handlePhase1bFromAcceptorShards([acceptors])"""
        return self.handlePhase1bFromAcceptorShards([acceptors], perm_seed=perm_seed)

    def handlePhase1bFromWire(self, decoder):
        """:159-191 over the Phase1bMessages of decoder's last decode (WireDecoder.decodeConsensusMessages), on the device;
        trigger_index is a message index of that decode (decoder.consensusValue(trigger_index) is cval as ids)"""
        o = self._p1_outs()
        N.check(N.lib().rapid_px_phase1b_wire(self._h, decoder._h, *[C.byref(x) for x in o]))
        return self._p1_result(o)

    @staticmethod
    def _p2_outs():
        return C.c_int32(0), C.c_int64(-1), C.c_uint64(0), C.c_uint64(0), C.c_int32(0)

    @staticmethod
    def _p2_result(o):
        d, i, a, b, l = o
        return Phase2bResult(bool(d.value), i.value, (a.value, b.value, l.value) if d.value else None)

    def handlePhase2bMessages(self, rnd, sender, value_hash, value_len, value_hash2=None, msg_cfg=None):
        """:223-236 over a batch in arrival order"""
        n = len(value_len)
        a0, a1 = _split_ranks(rnd, n)
        s = N.as_i32(sender)
        h1, ln = _u64(value_hash), N.as_i32(value_len)
        h2 = None if value_hash2 is None else _u64(value_hash2)
        mc = None if msg_cfg is None else N.as_i64(msg_cfg)
        o = self._p2_outs()
        N.check(N.lib().rapid_px_phase2b(self._h, n, N.ptr(mc), N.ptr(a0), N.ptr(a1), N.ptr(s), N.ptr(h1), N.ptr(h2), N.ptr(ln),
                                         *[C.byref(x) for x in o]))
        return self._p2_result(o)

    def handlePhase2bFromAcceptors(self, acceptors, perm_seed=0):
        """the Phase2b broadcasts of one PaxosAcceptors: handlePhase2bFromAcceptorShards([acceptors])"""
        return self.handlePhase2bFromAcceptorShards([acceptors], perm_seed=perm_seed)

    def handlePhase2bFromWire(self, decoder):
        """:223-236 over the Phase2bMessages of decoder's last decode, on the device.  Raises RapidError(EINVAL), nothing
        changed, if a message of the current configuration comes from an endpoint outside the dictionary"""
        o = self._p2_outs()
        N.check(N.lib().rapid_px_phase2b_wire(self._h, decoder._h, *[C.byref(x) for x in o]))
        return self._p2_result(o)

    @staticmethod
    def _shard_handles(shards):
        return (C.c_void_p * max(len(shards), 1))(*[s._h.value for s in shards])

    def handlePhase1bFromAcceptorShards(self, shards, comm=None, perm_seed=0):
        """:159-191 over the Phase1b answers of the last handlePhase1aMessage of several PaxosAcceptors shards (any order,
        disjoint ranges), as one handle over their union would deliver them: in acceptor order (perm_seed == 0) or in a
        seeded permutation; with an NcclComm, a collective call over every rank's shards that gives every rank the same result"""
        o = self._p1_outs()
        N.check(N.lib().rapid_px_phase1b_from_acceptor_shards(self._h, self._shard_handles(shards), len(shards),
                                                              None if comm is None else comm._h, int(perm_seed),
                                                              *[C.byref(x) for x in o]))
        return self._p1_result(o)

    def handlePhase2bFromAcceptorShards(self, shards, comm=None, perm_seed=0):
        """:223-236 over the Phase2b broadcasts of the last handlePhase2aMessage of several PaxosAcceptors shards, as
        handlePhase1bFromAcceptorShards"""
        o = self._p2_outs()
        N.check(N.lib().rapid_px_phase2b_from_acceptor_shards(self._h, self._shard_handles(shards), len(shards),
                                                              None if comm is None else comm._h, int(perm_seed),
                                                              *[C.byref(x) for x in o]))
        return self._p2_result(o)

    def lastDeviceMs(self):
        out = C.c_float(0)
        N.check(N.lib().rapid_px_last_device_ms(self._h, C.byref(out)))
        return out.value


class PaxosAcceptors:
    """rnd / vrnd / vval (Paxos.java:63-65) of n_acceptors virtual nodes in HBM; acceptor r is node acceptor_begin + r."""

    def __init__(self, configuration_id, n_acceptors, acceptor_begin=0, device=0):
        self.cfg, self.R, self.begin = int(configuration_id), int(n_acceptors), int(acceptor_begin)
        self._h = C.c_void_p()
        N.check(N.lib().rapid_pxa_create(C.byref(self._h), self.cfg, self.R, self.begin, device))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            N.lib().rapid_pxa_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, configuration_id):
        self.cfg = int(configuration_id)
        N.check(N.lib().rapid_pxa_reset(self._h, self.cfg))

    def registerFastRoundVotes(self, acceptor, value_hash, value_len, value_hash2=None):
        """:244-257 for the listed acceptors, as one-by-one calls in list order: an acceptor listed twice keeps its last vote"""
        a = N.as_i64(acceptor)
        h1, ln = _u64(value_hash), N.as_i32(value_len)
        h2 = None if value_hash2 is None else _u64(value_hash2)
        N.check(N.lib().rapid_pxa_register_fast_round_votes(self._h, len(a), N.ptr(a), N.ptr(h1), N.ptr(h2), N.ptr(ln)))

    def registerFastRoundVotesFrom(self, cluster):
        """every receiver of a VirtualCluster that announced in its last batch registers its proposal (FastPaxos.propose :94-98)"""
        N.check(N.lib().rapid_pxa_register_fast_round_votes_cd(self._h, cluster._h))

    def handlePhase1aMessage(self, rank, msg_cfg=None):
        """:120-151 for one broadcast message -> number of Phase1bMessages sent back (kept on the device)"""
        out = C.c_int64(0)
        N.check(N.lib().rapid_pxa_phase1a(self._h, self.cfg if msg_cfg is None else int(msg_cfg), int(rank[0]), int(rank[1]), C.byref(out)))
        return out.value

    def handlePhase2aMessage(self, rnd, value, msg_cfg=None):
        """:198-216 for one broadcast message -> number of Phase2bMessages broadcast (kept on the device)"""
        out = C.c_int64(0)
        h1, h2, ln = value
        N.check(N.lib().rapid_pxa_phase2a(self._h, self.cfg if msg_cfg is None else int(msg_cfg), int(rnd[0]), int(rnd[1]), int(h1), int(h2),
                                          int(ln), C.byref(out)))
        return out.value

    def setSilent(self, silent=None):
        """acceptors with silent[r] != 0 (crashed processes) neither change nor answer in handlePhase1aMessage /
        handlePhase2aMessage; None: every acceptor answers again"""
        m = None if silent is None else N.as_u8(silent)
        assert m is None or len(m) == self.R
        N.check(N.lib().rapid_pxa_set_silent(self._h, N.ptr(m)))

    def findValue(self, value):
        """lowest acceptor index whose vval is value = (hash, hash2, len), -1 if none.  Finds a proposer of a decision when
        called before handlePhase2aMessage overwrites the vvals"""
        h1, h2, ln = value
        out = C.c_int64(-1)
        N.check(N.lib().rapid_pxa_find_value(self._h, int(h1), int(h2), int(ln), C.byref(out)))
        return out.value

    def read(self, acceptor):
        """-> {'rnd': (r, i), 'vrnd': (r, i), 'vval': (hash, hash2, len)}"""
        rk = np.zeros(4, np.int32)
        a, b, l = C.c_uint64(0), C.c_uint64(0), C.c_int32(0)
        N.check(N.lib().rapid_pxa_read(self._h, int(acceptor), N.ptr(rk), C.byref(a), C.byref(b), C.byref(l)))
        rk = rk.tolist()
        return {"rnd": (rk[0], rk[1]), "vrnd": (rk[2], rk[3]), "vval": (a.value, b.value, l.value)}
