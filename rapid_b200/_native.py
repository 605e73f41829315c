"""ctypes binding of librapid_b200.so — the C ABI declared in include/rapid_b200.h.

The library is the product; this module only loads it.  There is no Python/CPU fallback: if the shared
object is missing it is built with nvcc, and if that is impossible the import of the compute classes fails
loudly.
"""
import ctypes as C
import os

import numpy as np

from . import _build

OK = 0
EINVAL, ENOT_IN_RING, EALREADY_IN_RING, EUUID_SEEN, EHASH_COLLISION, ECUDA, ENCCL, ENOMEM, EUNSUPPORTED = range(-1, -10, -1)

CD_SERVICE, CD_RAW, CD_SWEEP, CD_BUCKETED, CD_LOG = 0, 1, 2, 4, 8
DELIVERY_BLOCKED, DELIVERY_BITMAP, DELIVERY_PERMUTED, DELIVERY_SHUFFLED_BATCHES = 1, 2, 4, 8
WIRE_REQUEST = 1
WIRE_FAST_ROUND_PHASE2B, WIRE_PHASE1A, WIRE_PHASE1B, WIRE_PHASE2A, WIRE_PHASE2B = 5, 6, 7, 8, 9   # RapidRequest cases
EDGE_UP, EDGE_DOWN = 0, 1
MAX_K = 14


class RapidError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("rapid_b200 error %d: %s" % (code, msg))
        self.code = code


class NodeNotInRingException(RapidError):
    """MembershipView.NodeNotInRingException (MembershipView.java:508-512)"""


class NodeAlreadyInRingException(RapidError):
    """MembershipView.NodeAlreadyInRingException (MembershipView.java:502-506)"""


class UUIDAlreadySeenException(RapidError):
    """MembershipView.UUIDAlreadySeenException (MembershipView.java:514-519)"""


class HashCollisionError(RapidError):
    pass


class Delivery(C.Structure):
    _fields_ = [("flags", C.c_uint32), ("blocked", C.c_void_p), ("bitmap", C.c_void_p), ("perm_seed", C.c_uint64)]


_LIB = None

_vp, _i32, _i64, _u32, _u64, _p = C.c_void_p, C.c_int32, C.c_int64, C.c_uint32, C.c_uint64, C.c_void_p
_pp = C.POINTER(C.c_void_p)

# name -> argtypes (every function returns int32 except rapid_version)
SIGNATURES = {
    "rapid_last_error": [C.c_char_p, C.c_size_t],
    "rapid_device_count": [_p],
    "rapid_view_create": [_pp, _i32, _i64, _p, _p, _p, _i32],
    "rapid_view_destroy": [_vp],
    "rapid_view_size": [_vp, _p],
    "rapid_view_ring": [_vp, _i32, _p],
    "rapid_view_keys": [_vp, _i32, _p],
    "rapid_view_observers": [_vp, _i32, _p, _p],
    "rapid_view_subjects": [_vp, _i32, _p, _p],
    "rapid_view_expected_observers": [_vp, _p, _i32, _i32, _p, _p],
    "rapid_view_ring_numbers": [_vp, _i32, _i32, _p],
    "rapid_view_tables": [_vp, _p, _p],
    "rapid_view_config_id": [_vp, _p, _p, _i64, _p],
    "rapid_view_register_joiners": [_vp, _i64, _p, _p, _p, _p],
    "rapid_view_num_joiners": [_vp, _p],
    "rapid_view_joiner_tables": [_vp, _p],
    "rapid_view_apply_cut": [_vp, _p, _i64, _p],
    "rapid_view_set_node_ids": [_vp, _p, _p],
    "rapid_view_set_joiner_ids": [_vp, _i32, _i64, _p, _p],
    "rapid_view_current_config_id": [_vp, _p],
    "rapid_view_overlay_spectrum": [_vp, _u64, C.c_double, _i32, _p, _p, _p, _p, _p],
    "rapid_cd_debug_stats": [_vp, _p, _p, _p, _p],
    "rapid_cd_debug_grid": [_vp, _p, _p],
    "rapid_cd_create": [_pp, _vp, _i32, _i32, _i64, _i64, _u32, _i64],
    "rapid_cd_destroy": [_vp],
    "rapid_cd_apply_batch": [_vp, _i64, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "rapid_cd_apply_batch_dev": [_vp, _i64, _i64, _p, _p, _p, _p, _p, _p],
    "rapid_cd_apply_batch_dev_async": [_vp, _i64, _i64, _p, _p, _p, _p, _p, _p],
    "rapid_cd_sync": [_vp],
    "rapid_cd_apply_batches": [_vp, _i64, _i64, _p, _p, _p, _p, _p, _i64, _p, _p, _p, _p, _p, _p, _p],
    "rapid_cd_apply_batches_dev": [_vp, _i64, _i64, _p, _p, _p, _p, _p, _i64, _p, _p],
    "rapid_cd_read_announced_in": [_vp, _p],
    "rapid_cd_sequence_stats": [_vp, _p, _p, _p, _p],
    "rapid_cd_read_outputs": [_vp, _p, _p, _p, _p],
    "rapid_cd_get_proposal": [_vp, _i64, _p, _i32, _p],
    "rapid_cd_num_proposals": [_vp, _i64, _p],
    "rapid_cd_proposal_census": [_vp, _p, _i32, _p, _p],
    "rapid_cd_read_census": [_vp, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "rapid_cd_census_classes_dev": [_vp, _p],
    "rapid_cd_read_census_classes": [_vp, _p],
    "rapid_cd_clear": [_vp],
    "rapid_cd_debug_masks": [_vp, _i64, _p, _p, _i32, _p],
    "rapid_cd_debug_counters": [_vp, _i64, _p, _p],
    "rapid_cd_last_path": [_vp, _p, _p],
    "rapid_cd_aggregate": [_vp, _i64, _p, _p, _p, _p, _i64, _p, _i32, _p],
    "rapid_cd_invalidate": [_vp, _i64, _p, _i32, _p],
    "rapid_proposal_fingerprint": [_p, _i64, _p, _p],
    "rapid_fp_create": [_pp, _i64, _i64, _i64, _i32],
    "rapid_fp_destroy": [_vp],
    "rapid_fp_reset": [_vp, _i64, _i64],
    "rapid_fp_tally": [_vp, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "rapid_fp_tally_cd": [_vp, _vp, _vp, _p, _p, _p, _p, _p, _p],
    "rapid_fp_epoch_async": [_vp, _vp, _vp, _i64, _i64, _i64, _p, _p, _p, _p, _p],
    "rapid_fp_tally_cd_async": [_vp, _vp, _vp],
    "rapid_fp_result": [_vp, _p, _p, _p, _p, _p, _p, _p],
    "rapid_fp_quorum": [_i64, _p],
    "rapid_cd_timer_start": [_vp],
    "rapid_fp_timer_stop": [_vp, _vp, _p],
    "rapid_comm_unique_id": [_p],
    "rapid_comm_init": [_pp, _i32, _i32, _p, _i32],
    "rapid_comm_destroy": [_vp],
    "rapid_cd_last_device_ms": [_vp, _p, _p],
    "rapid_fp_last_device_ms": [_vp, _p],
    "rapid_fp_last_launches": [_vp, _p],
    "rapid_px_create": [_pp, _i64, _i64, _i64, _i32],
    "rapid_px_destroy": [_vp],
    "rapid_px_reset": [_vp, _i64, _i64],
    "rapid_pxa_reset": [_vp, _i64],
    "rapid_wire_create": [_pp, _vp],
    "rapid_wire_destroy": [_vp],
    "rapid_wire_set_configuration": [_vp, _i64],
    "rapid_wire_decode_alerts": [_vp, _p, _i64, _u32, _p, _p, _p, _p, _p],
    "rapid_wire_cells_dev": [_vp, _p, _p, _p, _p, _p],
    "rapid_wire_read_cells": [_vp, _p, _p, _p, _p, _p],
    "rapid_wire_read_messages": [_vp, _p, _p, _p, _p, _p, _p, _p, _p],
    "rapid_wire_decode_votes": [_vp, _p, _p, _i64, _u32, _p, _p, _p, _p, _p],
    "rapid_wire_last_device_ms": [_vp, _p],
    "rapid_wire_decode_consensus": [_vp, _i32, _p, _p, _i64, _u32, _p, _p],
    "rapid_wire_read_consensus": [_vp, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "rapid_wire_consensus_value": [_vp, _i64, _p, _i32, _p],
    "rapid_px_phase1b_wire": [_vp, _vp, _p, _p, _p, _p, _p, _p],
    "rapid_px_phase2b_wire": [_vp, _vp, _p, _p, _p, _p, _p],
    "rapid_fp_tally_wire": [_vp, _vp, _p, _p, _p, _p, _p, _p],
    "rapid_wire_encode_alert_batches": [_vp, _vp, _u32, _p, _p],
    "rapid_wire_encode_votes": [_vp, _vp, _i64, _u32, _p, _p],
    "rapid_wire_encoded_counts": [_vp, _p, _p, _p, _p],
    "rapid_wire_encoded_dev": [_vp, _p, _p, _p, _p, _p],
    "rapid_wire_read_encoded": [_vp, _p, _p, _p, _p, _p],
    "rapid_wire_read_encoded_sizes": [_vp, _p],
    "rapid_wire_encode_phase1b": [_vp, _vp, _vp, _u32, _p, _p],
    "rapid_wire_encode_phase2b": [_vp, _vp, _vp, _u32, _p, _p],
    "rapid_wire_read_encoded_senders": [_vp, _p],
    "rapid_fdet_create": [_pp, _vp, _i32, _i32],
    "rapid_fdet_destroy": [_vp],
    "rapid_fdet_reset": [_vp],
    "rapid_fdet_tick": [_vp, _p, _p, _i64, _p, _p],
    "rapid_fdet_tick_dev": [_vp, _p, _p, _i64, _p, _p],
    "rapid_fdet_cells_dev": [_vp, _p, _p, _p, _p, _p],
    "rapid_fdet_sender_batches": [_vp, _p, _i64, _p],
    "rapid_fdet_join_alerts": [_vp, _p, _i64, _i64, _p, _p],
    "rapid_fdet_merge_alerts": [_vp, _p, _i64, _p, _i64, _i64, _p, _p],
    "rapid_fdet_read_cells": [_vp, _p, _p, _p, _p, _p],
    "rapid_fdet_read_alerts": [_vp, _p, _p, _p],
    "rapid_fdet_state": [_vp, _i64, _i32, _p, _p],
    "rapid_fdet_last_device_ms": [_vp, _p],
    "rapid_px_start_phase1a": [_vp, _i32, _i32, _p],
    "rapid_px_coordinator_rule": [_vp, _i64, _p, _p, _p, _p, _p, _p],
    "rapid_px_phase1b": [_vp, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "rapid_px_phase2b": [_vp, _i64, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p],
    "rapid_px_last_device_ms": [_vp, _p],
    "rapid_pxa_create": [_pp, _i64, _i64, _i64, _i32],
    "rapid_pxa_destroy": [_vp],
    "rapid_pxa_register_fast_round_votes": [_vp, _i64, _p, _p, _p, _p],
    "rapid_pxa_register_fast_round_votes_cd": [_vp, _vp],
    "rapid_pxa_phase1a": [_vp, _i64, _i32, _i32, _p],
    "rapid_pxa_phase2a": [_vp, _i64, _i32, _i32, _u64, _u64, _i32, _p],
    "rapid_px_phase1b_from_acceptor_shards": [_vp, _p, _i32, _vp, _u64, _p, _p, _p, _p, _p, _p],
    "rapid_px_phase2b_from_acceptor_shards": [_vp, _p, _i32, _vp, _u64, _p, _p, _p, _p, _p],
    "rapid_pxa_read": [_vp, _i64, _p, _p, _p, _p],
    "rapid_pxa_set_silent": [_vp, _p],
    "rapid_pxa_find_value": [_vp, _u64, _u64, _i32, _p],
}


def library_path():
    return _build.LIB


def lib():
    """Load (building first if needed) librapid_b200.so.  Raises if it cannot be had."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = _build.LIB
    if not os.path.exists(path):
        _build.build_native()
    L = C.CDLL(path)
    L.rapid_version.restype = C.c_char_p
    L.rapid_version.argtypes = []
    for name, args in SIGNATURES.items():
        f = getattr(L, name)     # AttributeError here == header/library mismatch: fail loudly
        f.restype = C.c_int32
        f.argtypes = args
    _LIB = L
    return L


def last_error():
    buf = C.create_string_buffer(512)
    lib().rapid_last_error(buf, 512)
    return buf.value.decode("utf-8", "replace")


_EXC = {ENOT_IN_RING: NodeNotInRingException, EALREADY_IN_RING: NodeAlreadyInRingException,
        EUUID_SEEN: UUIDAlreadySeenException, EHASH_COLLISION: HashCollisionError}


def check(rc):
    if rc != OK:
        raise _EXC.get(rc, RapidError)(rc, last_error())


def ptr(a):
    """host pointer of a numpy array (None -> NULL)"""
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def device_count():
    n = C.c_int32(0)
    rc = lib().rapid_device_count(C.byref(n))
    return n.value if rc == OK else 0


def as_i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def as_u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


def as_i64(a):
    return np.ascontiguousarray(a, dtype=np.int64)


def pack_hostnames(hostnames):
    """list of str/bytes -> (uint8 bytes, int32 offsets[n+1])"""
    bs = [h.encode("utf-8") if isinstance(h, str) else bytes(h) for h in hostnames]
    off = np.zeros(len(bs) + 1, np.int32)
    if bs:
        off[1:] = np.cumsum([len(b) for b in bs])
    joined = b"".join(bs)
    hb = np.frombuffer(joined, dtype=np.uint8).copy() if joined else np.zeros(1, np.uint8)
    return hb, off
