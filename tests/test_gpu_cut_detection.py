"""The cut-detection kernels vs the oracle, through the C ABI.

First the reference's own CutDetectionTest (rapid/src/test/java/com/vrg/rapid/CutDetectionTest.java) driven through
RAW handles; then the MembershipService batch semantics for R virtual nodes on the BASELINE configs' shapes."""
import numpy as np
import pytest

from helpers import OracleWorld, compare_batch, random_batch
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu
K, H, L = 10, 8, 2
UP, DOWN = 0, 1
CFG = -1


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.fixture()
def view30(rb):
    # 127.0.0.2:2..31 are the subjects the Java tests use; sources are arbitrary ids (src is never read back)
    return rb.MembershipView(K, ["127.0.0.2"] * 30, list(range(2, 32)))


def test_cut_detection(rb, view30):                        # CutDetectionTest.java:43-59
    wb = rb.MultiNodeCutDetector(view30, H, L)
    dst = 0
    for i in range(H - 1):
        assert wb.aggregateForProposal(i + 1, dst, UP, i) == [] and wb.getNumProposals() == 0
    assert wb.aggregateForProposal(H, dst, UP, H - 1) == [dst] and wb.getNumProposals() == 1


def test_blocking_one_blocker(rb, view30):                 # :62-91
    wb = rb.MultiNodeCutDetector(view30, H, L)
    for d in (0, 1):
        for i in range(H - 1):
            assert wb.aggregateForProposal(i + 1, d, UP, i) == [] and wb.getNumProposals() == 0
    assert wb.aggregateForProposal(H, 0, UP, H - 1) == [] and wb.getNumProposals() == 0
    assert wb.aggregateForProposal(H, 1, UP, H - 1) == [0, 1] and wb.getNumProposals() == 1


def test_blocking_three_blockers(rb, view30):              # :95-137
    wb = rb.MultiNodeCutDetector(view30, H, L)
    for d in (0, 1, 2):
        for i in range(H - 1):
            assert wb.aggregateForProposal(i + 1, d, UP, i) == []
    assert wb.aggregateForProposal(H, 0, UP, H - 1) == [] and wb.getNumProposals() == 0
    assert wb.aggregateForProposal(H, 2, UP, H - 1) == [] and wb.getNumProposals() == 0
    assert wb.aggregateForProposal(H, 1, UP, H - 1) == [0, 1, 2] and wb.getNumProposals() == 1


def test_blocking_multiple_blockers_past_h(rb, view30):    # :140-189
    wb = rb.MultiNodeCutDetector(view30, H, L)
    for d in (0, 1, 2):
        for i in range(H - 1):
            assert wb.aggregateForProposal(i + 1, d, UP, i) == []
    wb.aggregateForProposal(H, 0, UP, H - 1)
    assert wb.aggregateForProposal(H + 1, 0, UP, H - 1) == [] and wb.getNumProposals() == 0
    wb.aggregateForProposal(H, 2, UP, H - 1)
    assert wb.aggregateForProposal(H + 1, 2, UP, H - 1) == [] and wb.getNumProposals() == 0
    assert wb.aggregateForProposal(H, 1, UP, H - 1) == [0, 1, 2] and wb.getNumProposals() == 1


def test_below_l(rb, view30):                              # :192-230
    wb = rb.MultiNodeCutDetector(view30, H, L)
    for i in range(H - 1):
        assert wb.aggregateForProposal(i + 1, 0, UP, i) == []
    for i in range(L - 1):
        assert wb.aggregateForProposal(i + 1, 1, UP, i) == []
    for i in range(H - 1):
        assert wb.aggregateForProposal(i + 1, 2, UP, i) == []
    assert wb.aggregateForProposal(H, 0, UP, H - 1) == [] and wb.getNumProposals() == 0
    assert wb.aggregateForProposal(H, 2, UP, H - 1) == [0, 2] and wb.getNumProposals() == 1


def test_batch(rb, view30):                                # :234-252
    wb = rb.MultiNodeCutDetector(view30, H, L)
    proposal = []
    for e in (0, 1, 2):
        proposal += wb.aggregateForProposal(5, e, UP, list(range(K)))     # one AlertMessage with K ring numbers
    assert sorted(proposal) == [0, 1, 2]


def test_link_invalidation(rb, view30):                    # :255-301
    wb = rb.MultiNodeCutDetector(view30, H, L)
    dst = 0
    observers = view30.getObserversOf(dst)
    assert len(observers) == K
    for i in range(H - 1):
        assert wb.aggregateForProposal(observers[i], dst, DOWN, i) == [] and wb.getNumProposals() == 0
    failed = set()
    for i in range(H - 1, K):
        oo = view30.getObserversOf(observers[i])
        failed.add(observers[i])
        for j in range(K):
            assert wb.aggregateForProposal(oo[j], observers[i], DOWN, j) == [] and wb.getNumProposals() == 0
    ret = wb.invalidateFailingEdges()
    assert len(ret) == 4 and wb.getNumProposals() == 1
    assert set(ret) == failed | {dst}
    wb.clear()
    assert wb.getNumProposals() == 0 and wb.invalidateFailingEdges() == []


def test_ctor_validation_and_bad_cells(rb, view30):        # MultiNodeCutDetector.java:51-55
    for h, l in ((11, 2), (8, 9), (8, 0), (0, 0)):
        with pytest.raises(ValueError):
            rb.MultiNodeCutDetector(view30, h, l)
    small = rb.MembershipView(2, ["a"], [1])
    with pytest.raises(ValueError):
        rb.MultiNodeCutDetector(small, 2, 1)               # K < 3
    wb = rb.MultiNodeCutDetector(view30, H, L)
    with pytest.raises(rb.RapidError):
        wb.aggregateForProposal(1, 0, UP, K)               # ring number >= K
    with pytest.raises(rb.RapidError):
        wb.aggregateForProposal(1, 31, UP, 0)              # unknown endpoint id


# ------------------------------------------------------------------------------------------------------
# MembershipService batch semantics for R virtual nodes
# ------------------------------------------------------------------------------------------------------
KERNELS = ["sweep", "bucketed"]


def _worlds(orc, rb, n, n_joiners=0, Hh=9, Ll=4, kernel="sweep", R=None, begin=0, Kx=K):
    w = OracleWorld(orc, n, Kx, n_joiners=n_joiners)
    v = rb.MembershipView.from_packed(Kx, *w.member_packed())
    if n_joiners:
        v.registerJoiners(*w.joiner_endpoints())
    R = n if R is None else R
    sim = orc.ClusterSim(w.view, Kx, Hh, Ll, R, receiver_base=begin)
    cl = rb.VirtualCluster(v, Hh, Ll, n_receivers=R, receiver_begin=begin, kernel=kernel)
    return w, v, sim, cl


@pytest.mark.parametrize("kernel", KERNELS)
def test_c1_single_crash(orc, rb, kernel):
    w, v, sim, cl = _worlds(orc, rb, 50, kernel=kernel)
    obs, _ = v.tables()
    b = W.c1_single_crash(obs, 50)
    blocked = W.blocked_by_receiver(b.blocked, v.getRing(0), 0, 50)
    o_len, o_ann = compare_batch(rb, w, sim, cl, None, (b.src, b.dst, b.ring, b.status), blocked=blocked)
    assert (o_len[blocked == 0] == 1).all() and (o_len[blocked == 1] == 0).all()
    # a second batch is ignored by everyone who announced (MembershipService.java:318-319)
    compare_batch(rb, w, sim, cl, None, (b.src, b.dst, b.ring, b.status), blocked=blocked)


@pytest.mark.parametrize("kernel", KERNELS)
def test_c2_simultaneous_crash(orc, rb, kernel):
    n = 2000
    w, v, sim, cl = _worlds(orc, rb, n, kernel=kernel)
    obs, _ = v.tables()
    b = W.c2_simultaneous_crash(obs, n, 0.01)
    blocked = W.blocked_by_receiver(b.blocked, v.getRing(0), 0, n)
    o_len, _ = compare_batch(rb, w, sim, cl, None, (b.src, b.dst, b.ring, b.status), blocked=blocked)
    live = np.nonzero(blocked == 0)[0]
    assert (o_len[live] == 20).all()
    assert cl.getProposal(int(live[0])) and sorted(cl.getProposal(int(live[0]))) == b.expected_cut.tolist()


@pytest.mark.parametrize("kernel", KERNELS)
def test_c3_correlated_partition_needs_invalidation(orc, rb, kernel):
    n = 2000
    w, v, sim, cl = _worlds(orc, rb, n, kernel=kernel)
    obs, _ = v.tables()
    b = W.c3_correlated_partition(obs, v.getRing(0), n, 0.05)
    blocked = W.blocked_by_receiver(b.blocked, v.getRing(0), 0, n)
    o_len, _ = compare_batch(rb, w, sim, cl, None, (b.src, b.dst, b.ring, b.status), blocked=blocked)
    live = np.nonzero(blocked == 0)[0]
    assert (o_len[live] == 100).all()          # the whole arc, emitted by invalidateFailingEdges


@pytest.mark.parametrize("kernel", KERNELS)
def test_c5_churn_joins_and_leaves(orc, rb, kernel):
    n, nl, nj = 3000, 15, 15
    w, v, sim, cl = _worlds(orc, rb, n, n_joiners=nj, kernel=kernel)
    obs, _ = v.tables()
    b = W.c5_churn(obs, w.joiner_obs(), n, nl, nj)
    blocked = W.blocked_by_receiver(b.blocked, v.getRing(0), 0, n)
    o_len, _ = compare_batch(rb, w, sim, cl, None, (b.src, b.dst, b.ring, b.status), blocked=blocked)
    live = np.nonzero(blocked == 0)[0]
    assert (o_len[live] == nl + nj).all()
    assert sorted(cl.getProposal(int(live[3]))) == b.expected_cut.tolist()


@pytest.mark.parametrize("kernel", KERNELS)
def test_filter_rules(orc, rb, kernel):
    """cfg mismatch, UP about a member, DOWN about a non-member are dropped (MembershipService.java:644-675)"""
    n, nj = 300, 4
    w, v, sim, cl = _worlds(orc, rb, n, n_joiners=nj, kernel=kernel)
    rng = np.random.default_rng(5)
    src, dst, ring, status = random_batch(rng, n + nj, K, 12, 150, n)
    status = rng.integers(0, 2, size=len(dst)).astype(np.uint8)          # deliberately inconsistent
    cfg = w.view.getCurrentConfigurationId()
    cell_cfg = np.where(rng.random(len(dst)) < 0.2, cfg + 1, cfg).astype(np.int64)
    compare_batch(rb, w, sim, cl, cfg, (src, dst, ring, status), cell_cfg=cell_cfg)


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("seed", range(6))
def test_random_multi_batch_streams(orc, rb, kernel, seed):
    """several batches with duplicates, carried state between batches, every receiver the same order"""
    n, nj = 400, 6
    Hh, Ll = [(9, 4), (8, 2), (8, 3), (9, 3), (5, 5), (10, 1)][seed]
    w, v, sim, cl = _worlds(orc, rb, n, n_joiners=nj, Hh=Hh, Ll=Ll, kernel=kernel)
    rng = np.random.default_rng(100 + seed)
    for _ in range(6):
        src, dst, ring, status = random_batch(rng, n + nj, K, int(rng.integers(1, 9)), int(rng.integers(1, 60)), n)
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, status))
    cl.clear(); sim.reset()
    src, dst, ring, status = random_batch(rng, n + nj, K, 3, 40, n)
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, status))


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("seed", range(4))
def test_per_receiver_delivery_bitmap(orc, rb, kernel, seed):
    """receivers see different subsets (partitions): masks, pre-proposals and announcements diverge"""
    n = 257
    w, v, sim, cl = _worlds(orc, rb, n, kernel=kernel, Hh=8, Ll=3)
    rng = np.random.default_rng(900 + seed)
    words = (n + 31) // 32
    for _ in range(5):
        src, dst, ring, status = random_batch(rng, n, K, int(rng.integers(2, 7)), int(rng.integers(5, 70)), n)
        bitmap = rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
        if seed % 2:
            bitmap |= rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
        blocked = (rng.random(n) < 0.1).astype(np.uint8)
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), blocked=blocked, bitmap=bitmap)


@pytest.mark.parametrize("seed", range(4))
def test_per_receiver_permuted_order(orc, rb, seed):
    """every receiver applies the batch in its own order (the K,H,L sensitivity-study shape): bucketed kernels only"""
    n = 300
    w, v, sim, cl = _worlds(orc, rb, n, kernel="bucketed", Hh=8, Ll=3, R=200, begin=50)
    rng = np.random.default_rng(40 + seed)
    for t in range(4):
        src, dst, ring, status = random_batch(rng, n, K, int(rng.integers(2, 8)), int(rng.integers(10, 80)), n)
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), perm_seed=W.SEED + 2 + t)


def test_c4_flip_flop_stream(orc, rb):
    n = 1000
    w, v, sim, cl = _worlds(orc, rb, n, kernel="bucketed")
    obs, _ = v.tables()
    batches = W.c4_flip_flop_stream(obs, n, 0.01, T=8)
    blocked = W.blocked_by_receiver(batches[0].blocked, v.getRing(0), 0, n)
    announced_any = False
    for b in batches:
        o_len, o_ann = compare_batch(rb, w, sim, cl, None, (b.src, b.dst, b.ring, b.status), blocked=blocked,
                                     perm_seed=b.meta["perm_seed"])
        announced_any |= bool(o_ann.any())
    assert announced_any


def test_sweep_rejects_permuted(orc, rb):
    w, v, sim, cl = _worlds(orc, rb, 50, kernel="sweep")
    with pytest.raises(rb.RapidError):
        cl.handleBatch(1, [0], [1], [0], [DOWN], perm_seed=3)


def test_num_proposals_sweep(orc, rb):
    n = 200
    w, v, sim, cl = _worlds(orc, rb, n, kernel="sweep", Hh=8, Ll=2)
    rng = np.random.default_rng(3)
    src, dst, ring, status = random_batch(rng, n, K, 3, 60, n)
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, status))
    for r in (0, 57, n - 1):
        assert cl.getNumProposals(r) == sim.numProposals(r)


@pytest.mark.parametrize("seed", range(6))
def test_num_proposals_on_the_bucketed_kernels_by_replay(orc, rb, seed):
    """getNumProposals (MultiNodeCutDetector.java:62-66) on a bucketed handle created with RAPID_CD_LOG: the receiver asked about is
    replayed through the per-cell rule over the epoch's cell log — several batches, blocked receivers, permuted delivery, a
    sequence call, several emissions inside one batch (small H / L); after clear() the count starts over."""
    rng = np.random.default_rng(4100 + seed)
    n = int(rng.integers(40, 600))
    Hh, Ll = [(8, 2), (9, 4), (3, 1)][seed % 3]
    w = OracleWorld(orc, n, K)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    sim = orc.ClusterSim(w.view, K, Hh, Ll, n)
    cl = rb.VirtualCluster(v, Hh, Ll, kernel="bucketed", log=True)
    cfg = w.view.getCurrentConfigurationId()
    for epoch in range(2):
        for call in range(3):
            src, dst, ring, status = random_batch(rng, n, K, int(rng.integers(1, 7)), int(rng.integers(10, 90)), n)
            blocked = (rng.random(n) < 0.15).astype(np.uint8) if call == 1 else None
            perm = int(rng.integers(1, 2**60)) if (seed + call) % 2 else None
            if call == 2:
                A = len(dst)
                off = np.concatenate([[0], np.sort(rng.integers(0, A + 1, size=3)), [A]]).astype(np.int64)
                for b in range(len(off) - 1):
                    sl = slice(int(off[b]), int(off[b + 1]))
                    sim.apply_batch(src[sl], dst[sl], ring[sl], status[sl], np.full(sl.stop - sl.start, cfg, np.int64), blocked=blocked,
                                    perm_seed=None if perm is None else perm + b, threads=2)
                cl.handleBatches(cfg, src, dst, ring, status, off, blocked=blocked, perm_seed=perm)
            else:
                compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), blocked=blocked, perm_seed=perm)
            for r in rng.choice(n, size=6, replace=False).tolist():
                assert cl.getNumProposals(r) == sim.numProposals(r), "receiver %d after call %d" % (r, call)
        if (Hh, Ll) == (3, 1):
            assert max(sim.numProposals(r) for r in range(n)) >= 1      # (with H = 3 the random batches do emit)
        cl.clear(); sim.reset()
        assert cl.getNumProposals(0) == 0
    # without the log the bucketed kernels cannot answer
    plain = rb.VirtualCluster(v, Hh, Ll, kernel="bucketed")
    with pytest.raises(rb.RapidError):
        plain.getNumProposals(0)


@pytest.mark.parametrize("permuted", [False, True])
def test_mixed_receivers_take_the_interval_analysis(orc, rb, permuted):
    """a proposal is emitted early in the batch, then another subject enters the unstable band and stays there:
    neither "everything resolved" nor "nothing emitted" — the exact interval analysis must run and agree."""
    n = 300
    w, v, sim, cl = _worlds(orc, rb, n, kernel="bucketed", Hh=8, Ll=3)
    rng = np.random.default_rng(77)
    seen_mixed = 0
    for trial in range(12):
        cl.clear(); sim.reset()
        a, bsub, c = (int(x) for x in rng.choice(n, size=3, replace=False))
        cells = [(a, k) for k in range(8)] + [(bsub, k) for k in range(int(rng.integers(3, 7)))]
        if trial % 2:
            cells = [(c, k) for k in range(9)] + cells              # two emission points before the blocker
        if trial % 3 == 0:
            rng.shuffle(cells)
        dst = np.array([x[0] for x in cells], np.int32)
        ring = np.array([x[1] for x in cells], np.uint8)
        src = np.zeros(len(cells), np.int32)
        status = np.full(len(cells), DOWN, np.uint8)
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), perm_seed=(1234 + trial) if permuted else None)
        seen_mixed += cl.debugStats()[0]
    assert seen_mixed > 0


@pytest.mark.parametrize("permuted", [False, True])
def test_interval_analysis_then_invalidation(orc, rb, permuted):
    """explicit proposals early in the batch, then subjects stuck in the band whose observers are partly the subjects that
    already left: the implicit pass must not count edges from observers that are no longer in proposal U preProposal"""
    n = 40
    rng = np.random.default_rng(2024)
    total_mixed = 0
    for trial in range(30):
        Hh, Ll = [(9, 4), (8, 3), (7, 2)][trial % 3]
        w, v, sim, cl = _worlds(orc, rb, n, kernel="bucketed", Hh=Hh, Ll=Ll)
        obs, _ = v.tables()
        s = int(rng.integers(0, n))
        o = list(dict.fromkeys(obs[s].tolist()))                         # distinct observers of s
        rng.shuffle(o)
        early = o[: int(rng.integers(1, 4))]                             # leave explicitly, first
        band = o[len(early): len(early) + int(rng.integers(0, 4))]       # stay in the unstable band
        cells = []
        for e in early:
            cells += [(e, k) for k in rng.permutation(K)[: int(rng.integers(Hh, K + 1))]]
        if trial % 4 == 0:
            rng.shuffle(cells)
        late = [(s, k) for k in rng.permutation(K)[: int(rng.integers(Ll, Hh))]]
        for bnode in band:
            late += [(bnode, k) for k in rng.permutation(K)[: int(rng.integers(Ll, Hh))]]
        rng.shuffle(late)
        cells += late
        dst = np.array([c[0] for c in cells], np.int32)
        ring = np.array([c[1] for c in cells], np.uint8)
        compare_batch(rb, w, sim, cl, None, (np.zeros(len(cells), np.int32), dst, ring, np.full(len(cells), DOWN, np.uint8)),
                      perm_seed=(99 + trial) if permuted else None)
        total_mixed += cl.debugStats()[0]
        # a follow-up batch: announced receivers ignore it, the others carry their state
        src2, dst2, ring2, st2 = random_batch(rng, n, K, 4, 30, n)
        compare_batch(rb, w, sim, cl, None, (src2, dst2, ring2, st2), perm_seed=(7 + trial) if permuted else None)
    assert total_mixed > 0


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("Kx,Hx,Lx", [(3, 3, 1), (5, 4, 2), (14, 12, 5), (7, 7, 7)])
def test_other_ring_counts(orc, rb, kernel, Kx, Hx, Lx):
    """K is a parameter of the view, not a constant of the kernels (K_MIN = 3, up to RAPID_MAX_K = 14)"""
    n = 150
    w = OracleWorld(orc, n, Kx)
    v = rb.MembershipView.from_packed(Kx, *w.member_packed())
    sim = orc.ClusterSim(w.view, Kx, Hx, Lx, n)
    cl = rb.VirtualCluster(v, Hx, Lx, kernel=kernel)
    rng = np.random.default_rng(Kx * 100 + Hx)
    obs, _ = v.tables()
    np.testing.assert_array_equal(obs, w.tables()[0])
    for _ in range(4):
        src, dst, ring, status = random_batch(rng, n, Kx, int(rng.integers(1, 6)), int(rng.integers(5, 50)), n)
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, status))
    b = W.c2_simultaneous_crash(obs, n, 0.02)
    cl.clear(); sim.reset()
    compare_batch(rb, w, sim, cl, None, (b.src, b.dst, b.ring, b.status))


@pytest.mark.parametrize("kernel", KERNELS)
def test_joiners_registered_after_the_detector_exists(orc, rb, kernel):
    """the id space grows (rapid_view_register_joiners) while a detector is alive: its dictionaries must follow"""
    n = 120
    w = OracleWorld(orc, n, K, n_joiners=70)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    sim = orc.ClusterSim(w.view, K, 9, 4, n)
    cl = rb.VirtualCluster(v, 9, 4, kernel=kernel)
    hosts, ports = w.joiner_endpoints()
    rng = np.random.default_rng(1)
    src, dst, ring, status = random_batch(rng, n, K, 3, 20, n)
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, status))
    with pytest.raises(rb.RapidError):
        cl.handleBatch(1, [0], [n + 3], [0], [UP])                       # not registered yet
    v.registerJoiners(hosts[:10], ports[:10])
    v.registerJoiners(hosts[10:], ports[10:])                             # 70 joiners > the initial id capacity slack
    jo = w.joiner_obs()
    cells_dst, cells_ring = [], []
    for j in (0, 9, 10, 69):
        for k in range(K):
            cells_dst.append(n + j); cells_ring.append(k)
    order = rng.permutation(len(cells_dst))
    dst = np.array(cells_dst, np.int32)[order]; ring = np.array(cells_ring, np.uint8)[order]
    src = jo[dst - n, ring]
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, np.full(len(dst), UP, np.uint8)))


@pytest.mark.parametrize("kernel", KERNELS)
def test_long_segments_and_heavy_duplication(orc, rb, kernel):
    """hundreds of cells about one subject in one batch (the StaticFailureDetector re-fires every tick)"""
    n = 90
    w, v, sim, cl = _worlds(orc, rb, n, kernel=kernel, Hh=9, Ll=4)
    rng = np.random.default_rng(4)
    a, b2 = 7, 33
    dst = np.concatenate([np.full(400, a), np.full(150, b2), rng.integers(0, n, size=60)]).astype(np.int32)
    ring = rng.integers(0, K, size=len(dst)).astype(np.uint8)
    order = rng.permutation(len(dst))
    dst, ring = dst[order], ring[order]
    src = rng.integers(0, n, size=len(dst)).astype(np.int32)
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, np.full(len(dst), DOWN, np.uint8)))
    if kernel == "bucketed":
        cl.clear(); sim.reset()
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, np.full(len(dst), DOWN, np.uint8)), perm_seed=5)


@pytest.mark.parametrize("permuted", [False, True])
def test_explicit_part_only_is_what_get_proposal_lists(orc, rb, permuted):
    """A leaves in an explicit proposal, then X and one of its observers enter the unstable band: the invalidation pass
    raises X (implicit report from the observer) but the observer itself stays stuck, so nothing more is emitted and the
    announced proposal is exactly the explicit part {A} — which rapid_cd_get_proposal must still be able to list."""
    n = 60
    rng = np.random.default_rng(31)
    hits = 0
    for trial in range(24):
        Hh, Ll = (9, 4) if trial % 2 else (8, 3)
        w, v, sim, cl = _worlds(orc, rb, n, kernel="bucketed", Hh=Hh, Ll=Ll)
        obs, _ = v.tables()
        x = int(rng.integers(0, n))
        xo = obs[x].tolist()
        o1 = xo[int(rng.integers(0, K))]
        rings_x = [k for k in range(K) if xo[k] != o1][: Hh - 1]          # X ends one short of H, none of it via o1
        if len(rings_x) < Ll or o1 == x:
            continue
        a = int(rng.choice([i for i in range(n) if i not in (x, o1) and i not in xo and i not in obs[o1].tolist()]))
        first = [(a, int(k)) for k in rng.permutation(K)[:Hh]]
        late = [(x, k) for k in rings_x] + [(o1, int(k)) for k in rng.permutation(K)[: int(rng.integers(Ll, Hh))]]
        rng.shuffle(late)
        cells = first + late
        dst = np.array([c[0] for c in cells], np.int32); ring = np.array([c[1] for c in cells], np.uint8)
        o_len, o_ann = compare_batch(rb, w, sim, cl, None, (np.zeros(len(cells), np.int32), dst, ring, np.full(len(cells), DOWN, np.uint8)),
                                     perm_seed=(40 + trial) if permuted else None)
        if o_len.max() == 1 and o_len.min() == 1:
            hits += 1
            assert cl.getProposal(0) == [a] and cl.getProposal(n - 1) == [a]
            assert cl.debugStats()[0] == n                             # every receiver went through the interval analysis
        # the next batch is ignored by those who announced; the others carry on
        src2, dst2, ring2, st2 = random_batch(rng, n, K, 3, 25, n)
        compare_batch(rb, w, sim, cl, None, (src2, dst2, ring2, st2), perm_seed=(90 + trial) if permuted else None)
    assert hits > 0 or permuted          # with per-receiver orders A is not first everywhere; parity above is the point


@pytest.mark.parametrize("kernel", KERNELS)
def test_empty_and_fully_filtered_batches(orc, rb, kernel):
    """empty batch, a batch whose every cell is dropped by the filter, then real work, then an empty batch again"""
    n = 100
    w, v, sim, cl = _worlds(orc, rb, n, kernel=kernel)
    empty = (np.zeros(0, np.int32),) * 2 + (np.zeros(0, np.uint8),) * 2
    compare_batch(rb, w, sim, cl, None, empty)
    cfg = w.view.getCurrentConfigurationId()
    rng = np.random.default_rng(2)
    src, dst, ring, status = random_batch(rng, n, K, 4, 30, n)
    compare_batch(rb, w, sim, cl, cfg, (src, dst, ring, status), cell_cfg=np.full(len(dst), cfg + 7, np.int64))   # all stale
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, np.zeros(len(dst), np.uint8)))                            # UP about members
    assert cl.debugMasks(0) == {} or all(m == 0 for m in cl.debugMasks(0).values())
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, status))
    compare_batch(rb, w, sim, cl, None, empty)
    blocked_all = np.ones(n, np.uint8)
    compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), blocked=blocked_all)                            # nobody receives it


def test_single_receiver_and_tiny_views(orc, rb):
    """R = 1 (seam 1 sizes) and a 3-node view through the bucketed kernels"""
    for n in (3, 4, 11):
        w, v, sim, cl = _worlds(orc, rb, n, kernel="bucketed", R=1, begin=n - 1)
        rng = np.random.default_rng(n)
        for _ in range(3):
            src, dst, ring, status = random_batch(rng, n, K, min(n, 3), 25, n)
            compare_batch(rb, w, sim, cl, None, (src, dst, ring, status))


@pytest.mark.parametrize("seed", range(8))
def test_fuzz_all_delivery_modes_combined(orc, rb, seed):
    """random K/H/L, joiners, several batches, and blocked + per-receiver subsets + per-receiver orders all at once"""
    rng = np.random.default_rng(7000 + seed)
    Kx = int(rng.integers(3, 15))
    Hx = int(rng.integers(1, Kx + 1))
    Lx = int(rng.integers(1, Hx + 1))
    n, nj = int(rng.integers(20, 200)), int(rng.integers(0, 6))
    R = int(rng.integers(1, n + 1))
    begin = int(rng.integers(0, n - R + 1))
    w = OracleWorld(orc, n, Kx, n_joiners=nj)
    v = rb.MembershipView.from_packed(Kx, *w.member_packed())
    if nj:
        v.registerJoiners(*w.joiner_endpoints())
    sim = orc.ClusterSim(w.view, Kx, Hx, Lx, R, receiver_base=begin)
    cl = rb.VirtualCluster(v, Hx, Lx, n_receivers=R, receiver_begin=begin, kernel="bucketed")
    words = (R + 31) // 32
    for t in range(int(rng.integers(2, 7))):
        src, dst, ring, status = random_batch(rng, n + nj, Kx, int(rng.integers(1, 8)), int(rng.integers(1, 70)), n)
        kw = {}
        if rng.random() < 0.6:
            kw["blocked"] = (rng.random(R) < 0.15).astype(np.uint8)
        if rng.random() < 0.6:
            bm = rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
            bm |= rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
            kw["bitmap"] = bm
        if rng.random() < 0.6:
            kw["perm_seed"] = int(rng.integers(0, 2**62))
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), **kw)
        if rng.random() < 0.15:
            cl.clear(); sim.reset()


# (K, kernel, seed): the K = 10 bucketed seeds with H = 9, L = 4, then every K from 3 to 14 on both kernels with (H, L) drawn per
# case; (K + kernel index) % 4 picks the draw, so each kernel meets (K, K), (K, 1), (1, 1) and a random pair at several K
MID_SCALE = [(10, "bucketed", s) for s in range(3)] + \
    [(Kx, kernel, 0) for Kx in range(3, 15) for kernel in KERNELS if (Kx, kernel) != (10, "bucketed")]


@pytest.mark.parametrize("Kx,kernel,seed", MID_SCALE,
                         ids=[str(s) if (Kx, k) == (10, "bucketed") else "%d-%s-K%d" % (s, k, Kx) for Kx, k, s in MID_SCALE])
def test_fuzz_mid_scale_shards(orc, rb, Kx, kernel, seed):
    """the same fuzz at a size where a shard spans several 1024-receiver row tiles and chunks: 2,500-4,000 nodes, a
    receiver shard that starts mid-tile, several hundred cells per batch over a few dozen subjects, every delivery mode (the
    sweep kernel takes every one but per-receiver orders)"""
    if (Kx, kernel) == (10, "bucketed"):
        rng = np.random.default_rng(9000 + seed)
        Hx, Lx = 9, 4
    else:
        ki = KERNELS.index(kernel)
        rng = np.random.default_rng((9000, Kx, ki, seed))
        Hx = [Kx, Kx, 1, int(rng.integers(1, Kx + 1))][(Kx + ki) % 4]
        Lx = [Hx, 1, 1, int(rng.integers(1, Hx + 1))][(Kx + ki) % 4]
    n, nj = int(rng.integers(2500, 4000)), int(rng.integers(0, 20))
    R = int(rng.integers(1100, n))
    begin = int(rng.integers(0, n - R + 1))
    w = OracleWorld(orc, n, Kx, n_joiners=nj)
    v = rb.MembershipView.from_packed(Kx, *w.member_packed())
    if nj:
        v.registerJoiners(*w.joiner_endpoints())
    sim = orc.ClusterSim(w.view, Kx, Hx, Lx, R, receiver_base=begin)
    cl = rb.VirtualCluster(v, Hx, Lx, n_receivers=R, receiver_begin=begin, kernel=kernel)
    words = (R + 31) // 32
    for t in range(4):
        src, dst, ring, status = random_batch(rng, n + nj, Kx, int(rng.integers(5, 40)), int(rng.integers(100, 500)), n)
        kw = {}
        if t != 1:
            kw["blocked"] = (rng.random(R) < 0.1).astype(np.uint8)
        if t >= 2:
            bm = rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
            bm |= rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
            kw["bitmap"] = bm
        if t % 2 == 1:
            perm = int(rng.integers(1, 2**62))
            if kernel == "bucketed":
                kw["perm_seed"] = perm
        compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), **kw)


def _per_sender(src, dst, ring, status):
    """group cells into one batch per sender, senders in order of first appearance, cells in their original order"""
    order, seen = [], {}
    for i, s in enumerate(src.tolist()):
        if s not in seen:
            seen[s] = len(order)
            order.append([])
        order[seen[s]].append(i)
    idx = np.array([i for g in order for i in g], np.int64)
    off = np.zeros(len(order) + 1, np.int64)
    off[1:] = np.cumsum([len(g) for g in order])
    return src[idx], dst[idx], ring[idx], status[idx], off


def _oracle_sequence(sim, cfg, src, dst, ring, status, off, n, blocked=None, perm_seed=None):
    """the oracle handling the batches one by one -> (announced_in, length, ids per announcer, announced flags)"""
    want_len, want_in, want_ids, o_ann = np.zeros(n, np.int32), np.full(n, -1, np.int32), {}, None
    for b in range(len(off) - 1):
        sl = slice(int(off[b]), int(off[b + 1]))
        o_len, o_ann, o_ids, o_off = sim.apply_batch(src[sl], dst[sl], ring[sl], status[sl], np.full(sl.stop - sl.start, cfg, np.int64),
                                                     blocked=blocked, perm_seed=None if perm_seed is None else perm_seed + b, threads=2)
        for r in np.nonzero(o_len)[0]:
            assert want_in[r] == -1                                   # a receiver announces once per configuration
            want_in[r], want_len[r] = b, o_len[r]
            want_ids[int(r)] = o_ids[o_off[r]: o_off[r + 1]].tolist()
    return want_in, want_len, want_ids, o_ann


def _check_sequence(rb, cl, sim, res, ain, want_in, want_len, want_ids, o_ann, check_masks=True):
    np.testing.assert_array_equal(ain, want_in)
    np.testing.assert_array_equal(res.proposal_len, want_len)
    np.testing.assert_array_equal(res.announced, o_ann)
    for r, ids in want_ids.items():
        assert rb.proposal_fingerprint(ids) == (int(res.proposal_hash[r]), int(res.proposal_hash2[r])), "receiver %d" % r
    for r, ids in list(want_ids.items())[:6]:
        assert cl.getProposal(r) == ids
    if check_masks:
        live = np.nonzero(o_ann == 0)[0]
        for r in live[:: max(1, len(live) // 8)][:8]:
            for subj, m in cl.debugMasks(int(r)).items():
                assert sim.reportMask(int(r), int(subj)) == m, "mask of subject %d at receiver %d" % (subj, r)
            assert cl.debugCounters(int(r))[0] == sim.updatesInProgress(int(r))


# the sequence tests at other ring counts: (H, L) by seed parity, one pair with H = K; at these K the views are larger (900 to
# 3,000 nodes), so some cases span several 1024-receiver tiles
SEQ_K = (3, 8, 11, 14)
SEQ_HL = {3: ((3, 1), (2, 1)), 8: ((8, 3), (7, 2)), 11: ((10, 4), (11, 5)), 14: ((13, 5), (14, 6))}
PER_SENDER = [(10, kernel, s) for kernel in KERNELS for s in range(8)] + \
    [(Kx, kernel, s) for Kx in SEQ_K for kernel in KERNELS for s in range(2)]


@pytest.mark.parametrize("Kx,kernel,seed", PER_SENDER, ids=["%d-%s%s" % (s, k, "" if Kx == 10 else "-K%d" % Kx) for Kx, k, s in PER_SENDER])
def test_sequence_of_per_sender_batches_matches_sequential_handling(orc, rb, Kx, seed, kernel):
    """the reference's AlertBatcher sends one BatchedAlertMessage per observer; a receiver handles them one by one and stops
    at the first that yields a proposal.  One rapid_cd_apply_batches call == the oracle handling the batches one by one."""
    if Kx == 10:
        rng = np.random.default_rng(12000 + seed)
        n, nj = int(rng.integers(30, 400)), int(rng.integers(0, 5))
        Hh, Ll = (9, 4) if seed % 2 else (8, 3)
    else:
        rng = np.random.default_rng((12000, Kx, seed))
        n, nj = int(rng.integers(900, 3000)), int(rng.integers(0, 5))
        Hh, Ll = SEQ_HL[Kx][seed % 2]
    w, v, sim, cl = _worlds(orc, rb, n, n_joiners=nj, Hh=Hh, Ll=Ll, kernel=kernel, Kx=Kx)
    cfg = w.view.getCurrentConfigurationId()
    for call in range(3):
        src, dst, ring, status = random_batch(rng, n + nj, Kx, int(rng.integers(1, 6)), int(rng.integers(5, 120)), n)
        src, dst, ring, status, off = _per_sender(src, dst, ring, status)
        blocked = (rng.random(n) < 0.1).astype(np.uint8) if call == 1 else None
        want = _oracle_sequence(sim, cfg, src, dst, ring, status, off, n, blocked=blocked)
        res, ain = cl.handleBatches(cfg, src, dst, ring, status, off, blocked=blocked)
        _check_sequence(rb, cl, sim, res, ain, *want)


def test_per_sender_batches_can_differ_from_one_merged_batch(orc, rb):
    """two crashes whose alerts do not interleave: sender by sender the first cut is announced alone; merged, both go together"""
    n = 60
    w, v, sim, cl = _worlds(orc, rb, n, kernel="sweep")
    obs = w.tables()[0]
    cfg = w.view.getCurrentConfigurationId()
    cells = [(int(obs[s][r]), s, r, 1) for s in (5, 17) for r in range(K)]          # all of 5's reports, then all of 17's
    src, dst, ring, status = (np.array(x) for x in zip(*cells))
    off = np.arange(len(cells) + 1, dtype=np.int64)                                  # worst case: one batch per cell
    res, ain = cl.handleBatches(cfg, src, dst, ring, status, off)
    assert set(res.proposal_len.tolist()) == {1} and set(ain.tolist()) == {8}        # the 9th report (H = 9) of node 5, alone
    merged = rb.VirtualCluster(v, 9, 4, kernel="sweep").handleBatch(cfg, src, dst, ring, status)
    assert set(merged.proposal_len.tolist()) == {2}
    # the subject-bucketed kernels: the one-pass treatment must be REFUSED here (node 5's cut is emitted before the last batch) and
    # the batch-by-batch replay gives the sequential answer
    bk = rb.VirtualCluster(v, 9, 4, kernel="bucketed")
    res2, ain2 = bk.handleBatches(cfg, src, dst, ring, status, off)
    assert set(res2.proposal_len.tolist()) == {1} and set(ain2.tolist()) == {8}
    assert bk.sequenceStats() == (0, 1)


SEQ_FUZZ = [(10, mode, s) for s in range(10) for mode in ("uniform", "permuted")] + \
    [(Kx, mode, s) for Kx in SEQ_K for s in range(3) for mode in ("uniform", "permuted")]


@pytest.mark.parametrize("Kx,mode,seed", SEQ_FUZZ, ids=["%d-%s%s" % (s, m, "" if Kx == 10 else "-K%d" % Kx) for Kx, m, s in SEQ_FUZZ])
def test_sequences_on_the_bucketed_path_fuzz(orc, rb, Kx, seed, mode):
    """rapid_cd_apply_batches on bucketed handles: random streams cut into random batches (a few long ones, many tiny ones,
    empty ones), uniform or per-receiver permuted delivery, blocked receivers, state carried from call to call — against the
    oracle handling every batch on its own.  Both outcomes of the one-pass attempt occur (served in one pass / refused and
    replayed) and must be indistinguishable; past K = 10 (a hi byte per receiver) every case takes both."""
    if Kx == 10:
        rng = np.random.default_rng(77000 + seed)
        n, nj = int(rng.integers(60, 1500)), int(rng.integers(0, 6))
        Hh, Ll = (9, 4) if seed % 3 else (8, 2)
    else:
        rng = np.random.default_rng((77000, Kx, seed, mode == "permuted"))
        n, nj = int(rng.integers(900, 3000)), int(rng.integers(0, 6))
        Hh, Ll = SEQ_HL[Kx][seed % 2]
    w, v, sim, cl = _worlds(orc, rb, n, n_joiners=nj, Hh=Hh, Ll=Ll, kernel="bucketed", Kx=Kx)
    cfg = w.view.getCurrentConfigurationId()
    obs = w.tables()[0]
    for call in range(4):
        if call % 2 == 0:
            # crash-shaped: every observer of a few subjects reports, spread over the batches (long unstable intervals: the
            # one-pass premises usually hold)
            subj = rng.choice(n, size=int(rng.integers(2, 12)), replace=False)
            cells = [(int(obs[s][r]), int(s), r, 1) for s in subj for r in range(Kx) if rng.random() < 0.95]
            order = rng.permutation(len(cells))
            src, dst, ring, status = (np.array(x) for x in zip(*[cells[i] for i in order]))
            src, dst = src.astype(np.int32), dst.astype(np.int32)
            ring, status = ring.astype(np.uint8), status.astype(np.uint8)
        else:
            src, dst, ring, status = random_batch(rng, n + nj, Kx, int(rng.integers(1, 8)), int(rng.integers(5, 150)), n)
        A = len(dst)
        nb = int(rng.integers(2, 12))
        cuts = np.sort(rng.integers(0, A + 1, size=nb - 1))
        off = np.concatenate([[0], cuts, [A]]).astype(np.int64)        # empty batches happen
        blocked = (rng.random(n) < 0.1).astype(np.uint8) if call % 3 == 1 else None
        perm = int(rng.integers(1, 2**60)) if mode == "permuted" else None
        want = _oracle_sequence(sim, cfg, src, dst, ring, status, off, n, blocked=blocked, perm_seed=perm)
        res, ain = cl.handleBatches(cfg, src, dst, ring, status, off, blocked=blocked, perm_seed=perm)
        _check_sequence(rb, cl, sim, res, ain, *want)
    one_pass, replayed = cl.sequenceStats()
    assert one_pass + replayed >= 1
    if Kx > 10:
        assert one_pass >= 1, cl.sequenceRefusal()                     # the random calls were served in one pass
        # then one call the one-pass attempt must refuse: all of one crashed node's reports, then another's, one batch per cell,
        # so the first cut is emitted before the last batch; the batch-by-batch replay gives the sequential answer
        cl.clear(); sim.reset()
        cells = [(int(obs[x][r]), x, r, 1) for x in (5, 17) for r in range(Kx)]
        src, dst, ring, status = (np.array(c) for c in zip(*cells))
        src, dst, ring, status = src.astype(np.int32), dst.astype(np.int32), ring.astype(np.uint8), status.astype(np.uint8)
        off = np.arange(len(cells) + 1, dtype=np.int64)
        perm = int(rng.integers(1, 2**60)) if mode == "permuted" else None
        want = _oracle_sequence(sim, cfg, src, dst, ring, status, off, n, perm_seed=perm)
        before = cl.sequenceStats()
        res, ain = cl.handleBatches(cfg, src, dst, ring, status, off, perm_seed=perm)
        _check_sequence(rb, cl, sim, res, ain, *want)
        assert (ain >= 0).all() and (ain < len(cells) - 1).all()
        assert cl.sequenceStats() == (before[0], before[1] + 1)        # this call was refused and replayed


def test_sequence_stream_c4_in_one_pass(orc, rb):
    """BASELINE config 4's shape (flip-flop stream, 8 batches, duplicates, per-receiver permuted order) as ONE sequence call: served
    in one pass over the state, same announcements as eight separate batches."""
    n = 3000
    w, v, sim, cl = _worlds(orc, rb, n, kernel="bucketed")
    cfg = w.view.getCurrentConfigurationId()
    obs = w.tables()[0]
    batches = W.c4_flip_flop_stream(obs, n, 0.01, T=8)
    blocked = W.blocked_by_receiver(batches[0].blocked, v.getRing(0), 0, n)
    src = np.concatenate([b.src for b in batches]); dst = np.concatenate([b.dst for b in batches])
    ring = np.concatenate([b.ring for b in batches]); status = np.concatenate([b.status for b in batches])
    off = np.concatenate([[0], np.cumsum([len(b) for b in batches])]).astype(np.int64)
    perm = batches[0].meta["perm_seed"]
    assert [b.meta["perm_seed"] for b in batches] == [perm + t for t in range(8)]
    want = _oracle_sequence(sim, cfg, src, dst, ring, status, off, n, blocked=blocked, perm_seed=perm)
    res, ain = cl.handleBatches(cfg, src, dst, ring, status, off, blocked=blocked, perm_seed=perm)
    _check_sequence(rb, cl, sim, res, ain, *want)
    live = blocked == 0
    assert (ain[live] == 7).all() and (res.proposal_len[live] == len(batches[-1].expected_cut)).all()
    assert cl.sequenceStats() == (1, 0), cl.sequenceRefusal()
    fp = rb.FastPaxos(cfg, n)
    t = fp.tallyCluster(cl)
    assert t.decided and t.length == len(batches[-1].expected_cut) and t.count == rb.quorum(n)
