"""GPU parity of alert generation (csrc/fd.cu, through the C ABI) against oracle::FdNode / PingPongFailureDetector: the
alerts of every interval, in order, under random crash / partition / bootstrapping / per-edge scenarios; then the whole
chain on the device — detectors -> cells -> cut detector -> the crashed set."""
import numpy as np
import pytest

from helpers import OracleWorld
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


# seeds 0-7 draw K from 3..12; three more seeds fix it at the smallest ring count and at the two largest (each draws a
# 300-node view)
INTERVAL_CASES = [(s, None) for s in range(8)] + [(13, 3), (9, 13), (10, 14)]


@pytest.mark.parametrize("seed,Kx", INTERVAL_CASES, ids=[str(s) if k is None else "%d-K%d" % (s, k) for s, k in INTERVAL_CASES])
def test_every_interval_matches_the_oracle(orc, rb, seed, Kx):
    rng = np.random.default_rng(seed)
    K = int(rng.integers(3, 13))
    if Kx is not None:
        K = Kx
    n = int(rng.choice([2, 3, 5, 8, 40, 300]))                 # tiny views: one subject on several rings
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    sim = orc.FdSim(w.view, K, np.arange(n))
    fd = rb.EdgeFailureDetectors(v)
    flags = np.zeros(n, np.uint8)
    edge = np.zeros(n * K, np.uint8)
    total = 0
    for t in range(60):
        if t % 7 == 0:                                        # the scenario drifts: nodes crash, partitions come and go
            flags = (rng.random(n) < 0.15).astype(np.uint8) * rng.choice([1, 2, 4, 8], n).astype(np.uint8)
            if rng.random() < 0.3:
                flags |= (rng.random(n) < 0.1).astype(np.uint8) * np.uint8(2)
            edge = (rng.random(n * K) < 0.05).astype(np.uint8)
        use_edge = t % 3 != 0
        want = sim.tick(flags, 11, edge if use_edge else None)
        na, nc = fd.tick(flags, 11, edge if use_edge else None)
        got = fd.alerts()
        assert got == want, "interval %d" % t
        assert na == len(want) and nc == sum(len(r) for _, _, r in want)
        src, dst, ring, status, cfg = fd.cells()
        assert list(zip(src.tolist(), dst.tolist(), ring.tolist())) == [(o, s, r) for o, s, rings in want for r in rings]
        assert (status == 1).all() and (cfg == 11).all()
        total += na
    assert total > 0 or n < 3
    for i in range(0, n, max(1, n // 7)):
        for k in range(sim.numDetectors(i)):
            assert fd.state(i, k) == sim.state(i, k)


def test_single_node_view_has_no_detectors(rb):
    hb, off, ports = W.packed_endpoints(0, 1)
    v = rb.MembershipView.from_packed(10, hb, off, ports)
    fd = rb.EdgeFailureDetectors(v)
    assert fd.tick(np.zeros(1, np.uint8), 1) == (0, 0)


def test_detectors_to_decision_without_leaving_the_device(orc, rb):
    """1 % of 20,000 nodes crash; eleven intervals later every live observer has raised its alerts; the cells go from
    the detectors' buffers straight into the cut detector and every live receiver proposes exactly the crashed set"""
    import ctypes as C
    from rapid_b200 import _native as Nn
    n, K = 20_000, 10
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    obs, _ = v.tables()
    b = W.c2_simultaneous_crash(obs, n)
    flags = np.zeros(n, np.uint8)
    flags[np.asarray(b.expected_cut)] = 1
    fd = rb.EdgeFailureDetectors(v)
    for t in range(10):
        assert fd.tick(flags, 5) == (0, 0)
    na, nc = fd.tick(flags, 5)
    assert nc == len(b.dst)
    src, dst, ring, status, cfg = fd.cells()
    assert sorted(zip(src.tolist(), dst.tolist(), ring.tolist())) == sorted(zip(b.src.tolist(), b.dst.tolist(), b.ring.tolist()))
    cl = rb.VirtualCluster(v, 9, 4, kernel="bucketed")
    p = fd.cellsDevice()
    ring0 = np.asarray(v.getRing(0))
    blocked = np.ascontiguousarray(flags[ring0])               # crashed receivers get nothing (receiver r = ring-0 position r)
    import torch
    d_blocked = torch.from_numpy(blocked).cuda()
    dl = Nn.Delivery()
    dl.flags = Nn.DELIVERY_BLOCKED
    dl.blocked = d_blocked.data_ptr()
    Nn.check(Nn.lib().rapid_cd_apply_batch_dev(cl._h, 5, nc, p[0], p[1], p[2], p[3], p[4], C.byref(dl)))
    res = cl.readOutputs()
    h1, h2 = rb.proposal_fingerprint(b.expected_cut)
    live = blocked == 0
    assert (np.asarray(res.proposal_len)[live] == len(b.expected_cut)).all()
    assert (np.asarray(res.proposal_hash)[live] == h1).all() and (np.asarray(res.proposal_hash2)[live] == h2).all()
    assert fd.tick(flags, 5) == (0, 0)                        # notified once


def test_detectors_to_per_sender_batches_on_the_device(orc, rb):
    """the same scenario shipped the way the reference ships it: ONE BatchedAlertMessage per sender (AlertBatcher,
    MembershipService.java:613-637), handled one by one with the announcedProposal gating — as a single rapid_cd_apply_batches_dev
    call on the cells in the detectors' buffers.  Checked against the oracle handling every sender's batch on its own."""
    _per_sender_batches_on_the_device(orc, rb, 4_000, 10, 9, 4)


def test_detectors_to_per_sender_batches_at_fourteen_rings(orc, rb):
    """the same at K = 14, H = 12: the detectors' cells feed the kernels whose rows hold a hi byte per receiver"""
    _per_sender_batches_on_the_device(orc, rb, 4_000, 14, 12, 5)


def _per_sender_batches_on_the_device(orc, rb, n, K, H, L):
    import torch
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    obs, _ = v.tables()
    b = W.c2_simultaneous_crash(obs, n)
    flags = np.zeros(n, np.uint8)
    flags[np.asarray(b.expected_cut)] = 1
    fd = rb.EdgeFailureDetectors(v)
    cfg = w.view.getCurrentConfigurationId()
    for t in range(10):
        assert fd.tick(flags, cfg) == (0, 0)
    na, nc = fd.tick(flags, cfg)
    off = fd.senderBatches()
    src, dst, ring, status, ccfg = fd.cells()
    assert off[0] == 0 and off[-1] == nc and len(off) - 1 == len(np.unique(src))
    assert all(len(set(src[off[i]: off[i + 1]].tolist())) == 1 for i in range(len(off) - 1))
    ring0 = np.asarray(v.getRing(0))
    blocked = np.ascontiguousarray(flags[ring0])
    d_blocked = torch.from_numpy(blocked).cuda()
    cl = rb.VirtualCluster(v, H, L, kernel="bucketed")
    p = fd.cellsDevice()
    cl.handleBatchesDevice(cfg, nc, p[1], p[2], p[3], off, cell_cfg_dev=p[4], blocked_dev=d_blocked.data_ptr())
    res, ain = cl.readOutputs(), cl.readAnnouncedIn()
    # the oracle: every sender's batch on its own, in order
    sim = orc.ClusterSim(w.view, K, H, L, n)
    want_in, want_len = np.full(n, -1, np.int32), np.zeros(n, np.int32)
    for i in range(len(off) - 1):
        sl = slice(int(off[i]), int(off[i + 1]))
        o_len, o_ann, o_ids, o_off = sim.apply_batch(src[sl], dst[sl], ring[sl], status[sl], ccfg[sl], blocked=blocked, threads=4)
        for r in np.nonzero(o_len)[0]:
            want_in[r], want_len[r] = i, o_len[r]
    np.testing.assert_array_equal(ain, want_in)
    np.testing.assert_array_equal(res.proposal_len, want_len)
    np.testing.assert_array_equal(res.announced, o_ann)
    live = blocked == 0
    assert (want_len[live] > 0).all()


def test_view_change_requires_reset(orc, rb):
    n, K = 50, 10
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    fd = rb.EdgeFailureDetectors(v)
    flags = np.zeros(n, np.uint8)
    flags[3] = 1
    for _ in range(5):
        fd.tick(flags, 1)
    v.applyCut([3])
    with pytest.raises(rb.RapidError):
        fd.tick(np.zeros(n - 1, np.uint8), 2)
    fd.reset()
    assert fd.tick(np.zeros(n - 1, np.uint8), 2) == (0, 0) and fd.state(0, 0) == (0, False)


def test_one_million_nodes_interval(rb):
    n, K = 1_000_000, 10
    hb, off, ports = W.packed_endpoints(0, n)
    v = rb.MembershipView.from_packed(K, hb, off, ports)
    fd = rb.EdgeFailureDetectors(v)
    flags = np.zeros(n, np.uint8)
    flags[W.pick_smallest(n, n // 200, 7)] = 1                # 5,000 crashes
    for _ in range(10):
        assert fd.tick(flags, 3) == (0, 0)
    quiet_ms = fd.lastDeviceMs()
    na, nc = fd.tick(flags, 3)
    assert 5000 * K * 0.9 < nc <= 5000 * K and na <= nc       # a few observers crashed too
    print("interval over %d detectors: %.3f ms quiet, %.3f ms raising %d alerts" % (n * K, quiet_ms, fd.lastDeviceMs(), na))
