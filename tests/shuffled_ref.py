"""RAPID_DELIVERY_SHUFFLED_BATCHES restated for the tests (NOT a pytest module): the batch order P_g of include/rapid_b200.h
twice — vectorised in NumPy and in plain Python integers — and the delivery itself over the oracle's literal handlers.

apply_batches drives oracle ClusterSim's R AlertBatchHandlers (each one MembershipService.handleMessage, gating included) through
tests/oracle_walk.cpp: every receiver r walks the batches in its own order P_{receiver_base + r} (a third, C++ restatement) and
stops after the batch it announces in.  The C++ file is compiled with g++ on first use into the temporary directory (the tree
may be read-only), together with oracle/oracle_capi.cpp for the handle types oracle/oracle_py.py creates."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from rapid_b200 import workloads as W

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORACLE = os.path.join(os.path.dirname(_HERE), "oracle")
_WALK = None

_M64 = (1 << 64) - 1


def order_width(n):
    """w: the smallest integer >= 4 with 4^w >= n"""
    w = 4
    while 4 ** w < n:
        w += 1
    return w


def batch_orders(seed, g, n):
    """[len(g)][n] int64: row i is P_{g[i]}(0..n-1), vectorised"""
    g = np.asarray(g, np.uint64).reshape(-1)
    if n <= 1:
        return np.zeros((len(g), n), np.int64)
    w = order_width(n)
    m, ws = np.uint64((1 << w) - 1), np.uint64(w)
    with np.errstate(over="ignore"):
        key = W.splitmix64(np.uint64(seed & _M64) + g)[:, None]

    def E(v):
        a, b = v >> ws, v & m
        for i in range(4):
            a, b = b, a ^ (W.splitmix64(key ^ np.uint64((i + 1) << 58) ^ b) & m)
        return (a << ws) | b

    v = E(np.tile(np.arange(n, dtype=np.uint64), (len(g), 1)))
    bad = v >= np.uint64(n)
    while bad.any():
        v = np.where(bad, E(v), v)
        bad = v >= np.uint64(n)
    return v.astype(np.int64)


def _sm(x):
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def batch_order_plain(seed, g, n):
    """P_g(0..n-1) in plain Python integers, written from the header's pseudocode"""
    if n <= 1:
        return list(range(n))
    w = order_width(n)
    m = (1 << w) - 1
    key = _sm((seed + g) & _M64)

    def E(v):
        a, b = v >> w, v & m
        for i in range(4):
            a, b = b, a ^ (_sm(key ^ ((i + 1) << 58) ^ b) & m)
        return (a << w) | b

    out = []
    for j in range(n):
        v = E(j)
        while v >= n:
            v = E(v)
        out.append(v)
    return out


def _walk():
    global _WALK
    if _WALK is None:
        srcs = [os.path.join(_HERE, "oracle_walk.cpp")] + [os.path.join(_ORACLE, f) for f in
                                                           ("oracle_capi.cpp", "rapid_oracle.hpp", "paxos_oracle.hpp", "fd_oracle.hpp", "xxh64.h")]
        tag = hashlib.sha256(b"".join(open(f, "rb").read() for f in srcs)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), "rapid_b200_oracle_walk_%s_%d.so" % (tag, os.getuid()))
        if not os.path.exists(so):
            tmp = "%s.%d.tmp" % (so, os.getpid())
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-pthread", "-shared", "-o", tmp, srcs[0]])
            os.replace(tmp, so)
        L = C.CDLL(so)
        p, i64, u64, i32 = C.c_void_p, C.c_int64, C.c_uint64, C.c_int32
        L.wk_batch_order.restype = None
        L.wk_batch_order.argtypes = [u64, i64, i64, p]
        L.wk_apply_batches.restype = i64
        L.wk_apply_batches.argtypes = [p, i64, p, p, p, p, p, i64, p, p, u64, i64, i32, p, p, p, p, i64]
        _WALK = L
    return _WALK


def batch_order_oracle(seed, g, n):
    """P_g(0..n-1) from the C++ restatement next to the oracle (tests/oracle_walk.cpp)"""
    out = np.zeros(max(n, 1), np.int64)
    _walk().wk_batch_order(seed & _M64, int(g), int(n), out.ctypes.data)
    return out[:n].tolist()


def _ptr(a):
    return None if a is None else a.ctypes.data


def apply_batches(sim, src, dst, ring, status, cfg, batch_off, blocked=None, order_seed=0, receiver_base=0, threads=None):
    """the sequence delivered to every receiver of the oracle ClusterSim `sim` in its own batch order
    -> (out_len, announced, proposals, announced_in): the length and list of the proposal each receiver announced in this call
    (0 / None if none), announcedProposal after the call, and the index of the announcing batch (-1 if none)"""
    R = sim.R
    off = np.ascontiguousarray(batch_off, np.int64)
    n = len(off) - 1
    src, dst = np.ascontiguousarray(src, np.int32), np.ascontiguousarray(dst, np.int32)
    ring, status = np.ascontiguousarray(ring, np.uint8), np.ascontiguousarray(status, np.uint8)
    cfg = np.ascontiguousarray(np.broadcast_to(np.asarray(cfg, np.int64), dst.shape))
    bl = None if blocked is None else np.ascontiguousarray(blocked, np.uint8)
    out_len, out_ann, out_in = np.zeros(R, np.int32), np.zeros(R, np.uint8), np.zeros(R, np.int32)
    # a proposal holds subjects of this call and of earlier ones: every subject this sim was ever given bounds it
    sim._walk_subjects = getattr(sim, "_walk_subjects", set()) | set(np.unique(dst).tolist())
    ids = np.empty(max(1, R * len(sim._walk_subjects)), np.int32)
    w = _walk().wk_apply_batches(sim.h, len(dst), _ptr(src), _ptr(dst), _ptr(ring), _ptr(status), _ptr(cfg), n, _ptr(off), _ptr(bl),
                                 order_seed & _M64, int(receiver_base), threads or min(16, os.cpu_count() or 1), _ptr(out_len),
                                 _ptr(out_ann), _ptr(out_in), _ptr(ids), len(ids))
    assert w >= 0
    pos = np.concatenate([[0], np.cumsum(out_len)])
    props = [ids[pos[r]: pos[r + 1]].tolist() if out_len[r] else None for r in range(R)]
    return out_len, out_ann, props, out_in
