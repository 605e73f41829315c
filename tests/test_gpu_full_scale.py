"""BASELINE.json's full sizes on the GPU, checked through size-independent properties (the oracle cannot finish these sizes in
seconds): every live virtual node announces the SAME proposal, its fingerprint is the fingerprint of the injected cut, the
canonical list is sorted by the ring-0 key, a repeated batch is ignored (announcedProposal), the fast round decides that cut
with exactly quorum votes counted, and the sweep kernel agrees with the bucketed kernels on a slice of the receivers."""
import numpy as np
import pytest

from rapid_b200 import workloads as W
from helpers import fingerprints_from_oracle

pytestmark = pytest.mark.gpu
K, H, L = 10, 9, 4


def _view(rb, n, nj=0, Kx=K):
    hb, off, ports = W.packed_endpoints(0, n + nj)
    v = rb.MembershipView.from_packed(Kx, hb[: off[n]], off[: n + 1], ports[:n])
    if nj:
        hosts, jports = W.endpoints(n, nj)
        v.registerJoiners(hosts, jports)
    return v


SAMPLE = 256


def _oracle_view(orc, n, nj=0, Kx=K):
    hb, off, ports = W.packed_endpoints(0, n + nj)
    u = orc.Universe()
    tags = u.add_bulk(hb, off, ports)
    hi, lo = W.node_ids(0, n)
    return u, orc.MembershipView(u, Kx, tags[:n], hi, lo)


def _sampled_oracle_check(orc, rb, oview, cl, res, window_begin, batch, cfg, blocked, perm_seed=None, sim=None, khl=(K, H, L)):
    """Per-receiver parity AT FULL SCALE: a window of SAMPLE receivers is run through the literal oracle on the same batch and
    compared receiver by receiver (length, both fingerprint words, announced flag, canonical list of one announcer, report
    masks + updatesInProgress of a few receivers that have not announced)."""
    if sim is None:
        sim = orc.ClusterSim(oview, *khl, SAMPLE, receiver_base=cl.receiver_begin + window_begin)
    o_len, o_ann, o_ids, o_off = sim.apply_batch(batch.src, batch.dst, batch.ring, batch.status, np.full(len(batch), cfg, np.int64),
                                                 blocked=blocked[window_begin: window_begin + SAMPLE], perm_seed=perm_seed, threads=8)
    sl = slice(window_begin, window_begin + SAMPLE)
    np.testing.assert_array_equal(res.proposal_len[sl], o_len)
    np.testing.assert_array_equal(res.announced[sl], o_ann)
    e1, e2 = fingerprints_from_oracle(rb, o_len, o_ids, o_off)
    np.testing.assert_array_equal(res.proposal_hash[sl], e1)
    np.testing.assert_array_equal(res.proposal_hash2[sl], e2)
    who = np.nonzero(o_len)[0]
    if len(who):
        r = int(who[len(who) // 2])
        assert cl.getProposal(window_begin + r, cap=int(o_len[r]) + 8) == o_ids[o_off[r]: o_off[r + 1]].tolist()
    quiet = np.nonzero(o_ann == 0)[0]
    for r in quiet[:: max(1, len(quiet) // 3)][:3]:
        for subj, m in cl.debugMasks(int(window_begin + r)).items():
            assert sim.reportMask(int(r), int(subj)) == m, "mask of subject %d at receiver %d" % (subj, window_begin + r)
        assert cl.debugCounters(int(window_begin + r))[0] == sim.updatesInProgress(int(r))
    return sim


def _check_converged(rb, v, cl, b, cfg, blocked, perm_seed=None):
    n = v.n
    res = cl.handleBatch(cfg, None, b.dst, b.ring, b.status, blocked=blocked, perm_seed=perm_seed)
    live = blocked == 0
    want = rb.proposal_fingerprint(b.expected_cut)
    assert (res.proposal_len[live] == len(b.expected_cut)).all() and (res.proposal_len[~live] == 0).all()
    assert (res.proposal_hash[live] == np.uint64(want[0])).all() and (res.proposal_hash2[live] == np.uint64(want[1])).all()
    assert (res.announced[live] == 1).all() and (res.announced[~live] == 0).all()
    # checksum of checksums: every live node contributed the same fingerprint
    assert int(res.proposal_len.sum()) == int(live.sum()) * len(b.expected_cut)
    # canonical order = ring-0 key order (MembershipService.java:346-348)
    r0 = int(np.nonzero(live)[0][len(np.nonzero(live)[0]) // 2])
    prop = cl.getProposal(r0, cap=len(b.expected_cut) + 8)
    assert sorted(prop) == b.expected_cut.tolist()
    keys0 = v.keys(0)[np.asarray(prop)]
    assert (np.diff(keys0) > 0).all()
    # idempotence: the same batch again is ignored by everyone who announced
    again = cl.handleBatch(cfg, None, b.dst, b.ring, b.status, blocked=blocked, perm_seed=perm_seed)
    assert (again.proposal_len == 0).all() and (again.announced == res.announced).all()
    return res, want


def _c5(orc, rb, n, khl, windows):
    """the C5 batch (n / 200 crashes, n / 200 joins) over n receivers: converged, the uniform kernel, per-receiver oracle parity on
    the windows, and the fast round's decision -> (view, batch, cfg, blocked, outputs)"""
    Kx, Hx, Lx = khl
    nj = n // 200
    v = _view(rb, n, nj, Kx)
    obs, _ = v.tables()
    b = W.c5_churn(obs, v.joinerTables(), n, n // 200, nj)
    hi, lo = W.node_ids(0, n)
    cfg = v.getCurrentConfigurationId(hi, lo)
    ring0 = v.getRing(0)
    blocked = W.blocked_by_receiver(b.blocked, ring0, 0, n)
    cl = rb.VirtualCluster(v, Hx, Lx, max_subjects=len(b.expected_cut) + 64)
    res, want = _check_converged(rb, v, cl, b, cfg, blocked)
    assert cl.lastPath()[0] == 2                                   # the subject-bucketed uniform kernel served it
    _, oview = _oracle_view(orc, n, nj, Kx)
    assert oview.getCurrentConfigurationId() == cfg
    for w0 in windows:
        _sampled_oracle_check(orc, rb, oview, cl, res, w0, b, cfg, blocked, khl=khl)
    # fast round: the decision is that cut, taken at the quorum-th vote
    cl.clear()
    cl.handleBatch(cfg, None, b.dst, b.ring, b.status, blocked=blocked, read_outputs=False)
    fp = rb.FastPaxos(cfg, n)
    t = fp.tallyCluster(cl)
    assert t.decided and (t.hash, t.hash2, t.length) == (want[0], want[1], len(b.expected_cut))
    assert t.count == rb.quorum(n) == t.votes_received
    del cl
    return v, b, cfg, blocked, res


def test_c5_one_million_nodes(orc):
    import rapid_b200 as rb
    n = 1_000_000
    # per-receiver oracle parity on two windows of the million receivers (one of them straddling a 1024-receiver tile edge)
    v, b, cfg, blocked, res = _c5(orc, rb, n, (K, H, L), (1024 * 300 - 100, 987_654))
    # the per-cell sweep kernel on a slice of the receivers agrees bit for bit
    lo_r, cnt = 123_456, 4096
    sw = rb.VirtualCluster(v, H, L, n_receivers=cnt, receiver_begin=lo_r, kernel="sweep", max_subjects=len(b.expected_cut) + 64)
    r2 = sw.handleBatch(cfg, None, b.dst, b.ring, b.status, blocked=blocked[lo_r: lo_r + cnt])
    assert (r2.proposal_hash == res.proposal_hash[lo_r: lo_r + cnt]).all()
    assert (r2.proposal_len == res.proposal_len[lo_r: lo_r + cnt]).all()


@pytest.mark.parametrize("n,khl", [(100_000, (11, 11, 4)), (150_000, (14, 12, 5))], ids=["K11", "K14"])
def test_c5_past_ten_rings(orc, n, khl):
    """the C5 shape where the rows hold a hi byte per receiver (K > 10, 2 B per (subject, receiver)): windows across a tile edge
    and at the end of the receivers, the same final tally"""
    import rapid_b200 as rb
    _c5(orc, rb, n, khl, (1024 * 60 - 100, n - SAMPLE))


def test_c3_ten_thousand_nodes_correlated_partition(orc):
    import rapid_b200 as rb
    n = 10_000
    v = _view(rb, n)
    obs, _ = v.tables()
    ring0 = v.getRing(0)
    b = W.c3_correlated_partition(obs, ring0, n, 0.05)
    hi, lo = W.node_ids(0, n)
    cfg = v.getCurrentConfigurationId(hi, lo)
    blocked = W.blocked_by_receiver(b.blocked, ring0, 0, n)
    cl = rb.VirtualCluster(v, H, L)
    res, _ = _check_converged(rb, v, cl, b, cfg, blocked)
    assert cl.debugStats()[1] > 0                                   # the cut came out of invalidateFailingEdges
    _, oview = _oracle_view(orc, n)
    for w0 in (0, 5000 - 128, n - SAMPLE):                          # includes receivers inside and next to the partitioned arc
        _sampled_oracle_check(orc, rb, oview, cl, res, w0, b, cfg, blocked)
    fp = rb.FastPaxos(cfg, n)
    cl.clear()
    cl.handleBatch(cfg, None, b.dst, b.ring, b.status, blocked=blocked, read_outputs=False)
    t = fp.tallyCluster(cl)
    assert t.decided and t.length == 500 and t.count == rb.quorum(n)


@pytest.mark.parametrize("n", [63 * 1024, 70_000])
def test_c3_partition_on_both_sides_of_the_invalidation_split(orc, n):
    """k_inval_finalize2 splits a tile's work list over several blocks below 64 tiles of 1024 receivers and gives every tile one
    block from 64 tiles on: a C3 partition at 63 tiles and at 69, checked receiver by receiver on windows that straddle a tile
    edge and windows inside the partitioned arc"""
    import rapid_b200 as rb
    v = _view(rb, n)
    obs, _ = v.tables()
    ring0 = v.getRing(0)
    b = W.c3_correlated_partition(obs, ring0, n, 0.05)
    hi, lo = W.node_ids(0, n)
    cfg = v.getCurrentConfigurationId(hi, lo)
    blocked = W.blocked_by_receiver(b.blocked, ring0, 0, n)
    cl = rb.VirtualCluster(v, H, L)
    res, _ = _check_converged(rb, v, cl, b, cfg, blocked)
    assert cl.debugStats()[1] > 0                                   # the cut came out of invalidateFailingEdges
    start, count = b.meta["arc_start"], len(b.expected_cut)
    # receivers are ring-0 positions, so the arc is receivers start .. start + count: one window across its edge, two inside it
    inside = [(start + d) % n for d in (-SAMPLE // 2, SAMPLE, count // 2)]
    windows = [1024 * 31 - SAMPLE // 2, 1024 * 62 - SAMPLE // 3] + [w0 for w0 in inside if w0 + SAMPLE <= n]
    assert len(windows) >= 3
    _, oview = _oracle_view(orc, n)
    for w0 in windows:
        _sampled_oracle_check(orc, rb, oview, cl, res, w0, b, cfg, blocked)
    fp = rb.FastPaxos(cfg, n)
    cl.clear()
    cl.handleBatch(cfg, None, b.dst, b.ring, b.status, blocked=blocked, read_outputs=False)
    t = fp.tallyCluster(cl)
    assert t.decided and t.length == count and t.count == rb.quorum(n)


def test_c4_hundred_thousand_nodes_flip_flop_stream(orc):
    import rapid_b200 as rb
    n = 100_000
    v = _view(rb, n)
    obs, _ = v.tables()
    ring0 = v.getRing(0)
    batches = W.c4_flip_flop_stream(obs, n, 0.01, T=8)
    hi, lo = W.node_ids(0, n)
    cfg = v.getCurrentConfigurationId(hi, lo)
    blocked = W.blocked_by_receiver(batches[0].blocked, ring0, 0, n)
    cl = rb.VirtualCluster(v, H, L)
    fp = rb.FastPaxos(cfg, n)
    want = rb.proposal_fingerprint(batches[-1].expected_cut)
    decided = None
    _, oview = _oracle_view(orc, n)
    windows = (1024 * 40 - 128, 77_777)
    sims = {}
    for b in batches:
        res = cl.handleBatch(cfg, None, b.dst, b.ring, b.status, blocked=blocked, perm_seed=b.meta["perm_seed"])
        for w0 in windows:                                          # state carried: the same oracle instances follow the whole stream
            sims[w0] = _sampled_oracle_check(orc, rb, oview, cl, res, w0, b, cfg, blocked, perm_seed=b.meta["perm_seed"], sim=sims.get(w0))
        assert cl.lastPath()[0] == 4                                # per-receiver order, every cell to everyone: uniform kernel, moments on demand
        ann = res.proposal_len > 0
        # whoever announces in a batch announces a subset of the flapping nodes; once everything is in, the whole set
        assert (res.proposal_len[ann] <= len(batches[-1].expected_cut)).all()
        t = fp.tallyCluster(cl)
        if t.decided:
            decided = t
            break
    assert decided is not None and (decided.hash, decided.hash2) == want and decided.count == rb.quorum(n)


class _Cells:
    """a slice of a workload batch, shaped like one for _sampled_oracle_check"""

    def __init__(self, b, sl):
        self.src, self.dst, self.ring, self.status = b.src[sl], b.dst[sl], b.ring[sl], b.status[sl]

    def __len__(self):
        return len(self.dst)


def test_c5_carried_halves_as_the_benchmark_runs_them(orc):
    """bench.py's roofline_carried path: the C5 batch delivered as two halves with no clear() in between, so the second half
    read-modify-writes the rows the first wrote (memo, L2 prefetch).  The same oracle instances follow both halves on a window
    across a tile edge and a window holding blocked receivers; then the fast round decides the cut."""
    import rapid_b200 as rb
    n = 1_000_000
    nj = n // 200
    v = _view(rb, n, nj)
    obs, _ = v.tables()
    b = W.c5_churn(obs, v.joinerTables(), n, n // 200, nj)
    hi, lo = W.node_ids(0, n)
    cfg = v.getCurrentConfigurationId(hi, lo)
    blocked = W.blocked_by_receiver(b.blocked, v.getRing(0), 0, n)
    cl = rb.VirtualCluster(v, H, L, max_subjects=len(b.expected_cut) + 64)
    half = len(b) // 2
    first = np.nonzero(blocked)[0]
    windows = (1024 * 500 - 100, int(min(max(first[len(first) // 2] - SAMPLE // 2, 0), n - SAMPLE)))
    assert blocked[windows[1]: windows[1] + SAMPLE].any()
    _, oview = _oracle_view(orc, n, nj)
    sims = {}
    for sl in (slice(0, half), slice(half, len(b))):
        part = _Cells(b, sl)
        res = cl.handleBatch(cfg, None, part.dst, part.ring, part.status, blocked=blocked)
        assert cl.lastPath()[0] == 2
        for w0 in windows:
            sims[w0] = _sampled_oracle_check(orc, rb, oview, cl, res, w0, part, cfg, blocked, sim=sims.get(w0))
    live = blocked == 0
    assert (res.announced[live] == 1).all() and (res.announced[~live] == 0).all()
    want = rb.proposal_fingerprint(b.expected_cut)
    fp = rb.FastPaxos(cfg, n)
    t = fp.tallyCluster(cl)
    assert t.decided and (t.hash, t.hash2, t.length) == (want[0], want[1], len(b.expected_cut))


def test_c4_as_one_sequence_call(orc):
    """bench.py's default C4 stream: ONE rapid_cd_apply_batches call over 100,000 receivers (the SEQ kernels and k_seq_check at
    98 tiles), served in one pass, against the oracle handling every batch on its own on two windows"""
    import rapid_b200 as rb
    n = 100_000
    v = _view(rb, n)
    obs, _ = v.tables()
    ring0 = v.getRing(0)
    batches = W.c4_flip_flop_stream(obs, n, 0.01, T=8)
    hi, lo = W.node_ids(0, n)
    cfg = v.getCurrentConfigurationId(hi, lo)
    blocked = W.blocked_by_receiver(batches[0].blocked, ring0, 0, n)
    src = np.concatenate([x.src for x in batches]); dst = np.concatenate([x.dst for x in batches])
    ring = np.concatenate([x.ring for x in batches]); status = np.concatenate([x.status for x in batches])
    off = np.concatenate([[0], np.cumsum([len(x) for x in batches])]).astype(np.int64)
    perm = batches[0].meta["perm_seed"]
    cl = rb.VirtualCluster(v, H, L)
    res, ain = cl.handleBatches(cfg, None, dst, ring, status, off, blocked=blocked, perm_seed=perm)
    assert cl.sequenceStats() == (1, 0), cl.sequenceRefusal()
    _, oview = _oracle_view(orc, n)
    for w0 in (1024 * 40 - 128, 77_777):
        sl = slice(w0, w0 + SAMPLE)
        sim = orc.ClusterSim(oview, K, H, L, SAMPLE, receiver_base=w0)
        want_in, want_len = np.full(SAMPLE, -1, np.int32), np.zeros(SAMPLE, np.int32)
        want_h1, want_h2 = np.zeros(SAMPLE, np.uint64), np.zeros(SAMPLE, np.uint64)
        for t in range(len(batches)):
            c = slice(int(off[t]), int(off[t + 1]))
            o_len, o_ann, o_ids, o_off = sim.apply_batch(src[c], dst[c], ring[c], status[c], np.full(c.stop - c.start, cfg, np.int64),
                                                         blocked=blocked[sl], perm_seed=perm + t, threads=8)
            e1, e2 = fingerprints_from_oracle(rb, o_len, o_ids, o_off)
            now = o_len > 0
            want_in[now], want_len[now], want_h1[now], want_h2[now] = t, o_len[now], e1[now], e2[now]
        np.testing.assert_array_equal(ain[sl], want_in)
        np.testing.assert_array_equal(res.proposal_len[sl], want_len)
        np.testing.assert_array_equal(res.proposal_hash[sl], want_h1)
        np.testing.assert_array_equal(res.proposal_hash2[sl], want_h2)
        np.testing.assert_array_equal(res.announced[sl], o_ann)
        quiet = np.nonzero(o_ann == 0)[0]
        for r in quiet[:: max(1, len(quiet) // 3)][:3]:
            for subj, m in cl.debugMasks(int(w0 + r)).items():
                assert sim.reportMask(int(r), int(subj)) == m, "mask of subject %d at receiver %d" % (subj, w0 + r)
            assert cl.debugCounters(int(w0 + r))[0] == sim.updatesInProgress(int(r))
    live = blocked == 0
    assert (ain[live] == len(batches) - 1).all()
