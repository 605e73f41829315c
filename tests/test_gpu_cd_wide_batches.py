"""Batches that bring 65,536 subjects or more across a threshold, on the subject-bucketed kernels.

The per-receiver and per-chunk counters of the apply kernels (subjects crossing L / H, subjects touched in the unstable band,
subjects left in it) sum over every subject of a chunk, and the counters of the fresh subjects sum over the whole batch.  A
batch that moves 70,000 subjects must count 70,000 of them.  The subjects are joiners (UP alerts): no DOWN alert is ever seen,
so no invalidation pass adds reports and the expected counts are analytic — every receiver that gets the cells has 70,000
subjects in progress after the L batch and announces all 70,000 after the H batch.  A 16-receiver window is also run through
the literal oracle.

Every case runs at K = 10 (two hi bits per receiver in the rows); the default grid and the one-chunk case also run at K = 14 (a
hi byte per receiver, 2 B per (subject, receiver))."""
import numpy as np
import pytest

from helpers import OracleWorld, fingerprints_from_oracle
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu
KHL = {10: (9, 4), 14: (13, 5)}       # K -> (H, L)
N_MEMBERS = 100_000
N_WIDE = 70_000                       # subjects moved by one batch: more than 2^16
R, BEGIN = 1003, 40_000 + 300         # the handle: R not a multiple of 8, starting mid-tile of the ring
WINDOW = 16
W0 = R - WINDOW                       # the oracle's window ends with the tile's tail receivers
DUP_CELLS = 700_000                   # one subject reported again and again: the next batch's grid estimate is 1 subject


_WORLD = {}


@pytest.fixture(scope="module", autouse=True)
def _free_worlds():
    """the worlds (a 170,000-id view on the device, the oracle's, the cell arrays) live as long as this module's tests"""
    yield
    _WORLD.clear()


@pytest.fixture(scope="module")
def world(orc, _free_worlds):
    return _world(orc, 10)


def _world(orc, K):
    """the view, its joiners and the batches at K rings, built once per K"""
    if K not in _WORLD:
        _WORLD[K] = _build_world(orc, K)
    return _WORLD[K]


def _build_world(orc, K):
    import rapid_b200 as rb
    H, L = KHL[K]
    w = OracleWorld(orc, N_MEMBERS, K, n_joiners=N_WIDE + 1)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    v.registerJoiners(*w.joiner_endpoints())
    jobs = v.joinerTables()
    cfg = w.view.getCurrentConfigurationId()
    subjects = np.arange(N_MEMBERS, N_MEMBERS + N_WIDE, dtype=np.int32)
    rng = np.random.default_rng(65536)

    def cells(rings, subj=subjects):
        """every subject reported on `rings` by its expected observer, in a seeded shuffled order"""
        dst = np.repeat(subj, len(rings))
        ring = np.tile(np.asarray(rings, np.uint8), len(subj))
        src = jobs[dst - N_MEMBERS, ring].astype(np.int32)
        order = rng.permutation(len(dst))
        return src[order], dst[order].astype(np.int32), ring[order], np.full(len(dst), W.UP, np.uint8)

    extra = N_MEMBERS + N_WIDE                                       # the one subject of the duplicate-heavy batches
    dup = (np.full(DUP_CELLS, jobs[N_WIDE, 0], np.int32), np.full(DUP_CELLS, extra, np.int32),
           np.zeros(DUP_CELLS, np.uint8), np.full(DUP_CELLS, W.UP, np.uint8))
    return dict(rb=rb, w=w, v=v, K=K, H=H, L=L, cfg=cfg, subjects=subjects, low=cells(range(L)), high=cells(range(L, H)), dup=dup)


def _bitmap(A, n_recv, base, gets):
    """every cell reaches the receivers r (absolute handle index base + local) with gets(r); the same row for every cell"""
    words = (n_recv + 31) // 32
    row = np.zeros(words, np.uint32)
    for r in range(n_recv):
        if gets(base + r):
            row[r >> 5] |= np.uint32(1 << (r & 31))
    return np.broadcast_to(row, (A, words))


def _gets(r):
    return r % 5 != 2


class Case:
    def __init__(self, d, bitmap=False):
        rb = d["rb"]
        self.d, self.rb, self.bitmap = d, rb, bitmap
        self.cl = rb.VirtualCluster(d["v"], d["H"], d["L"], n_receivers=R, receiver_begin=BEGIN, kernel="bucketed",
                                    max_subjects=N_WIDE + 64)
        self.sim = d["w"].orc.ClusterSim(d["w"].view, d["K"], d["H"], d["L"], WINDOW, receiver_base=BEGIN + W0)
        self.want = rb.proposal_fingerprint(d["subjects"])

    def batch(self, arrays, oracle=True):
        src, dst, ring, status = arrays
        kw, okw = {}, {}
        if self.bitmap and oracle:
            kw["bitmap"] = _bitmap(len(dst), R, 0, _gets)
            okw["bitmap"] = _bitmap(len(dst), WINDOW, W0, _gets)
        res = self.cl.handleBatch(self.d["cfg"], src, dst, ring, status, **kw)
        if oracle:
            o_len, o_ann, o_ids, o_off = self.sim.apply_batch(src, dst, ring, status, np.full(len(dst), self.d["cfg"], np.int64),
                                                              threads=8, **okw)
            self.compare(res, o_len, o_ann, o_ids, o_off)
        return res

    def compare(self, res, o_len, o_ann, o_ids, o_off):
        sl = slice(W0, W0 + WINDOW)
        np.testing.assert_array_equal(res.proposal_len[sl], o_len)
        np.testing.assert_array_equal(res.announced[sl], o_ann)
        e1, e2 = fingerprints_from_oracle(self.rb, o_len, o_ids, o_off)
        np.testing.assert_array_equal(res.proposal_hash[sl], e1)
        np.testing.assert_array_equal(res.proposal_hash2[sl], e2)
        who = np.nonzero(o_len)[0]
        if len(who):
            r = int(who[len(who) // 2])
            assert self.cl.getProposal(W0 + r, cap=N_WIDE + 8) == o_ids[o_off[r]: o_off[r + 1]].tolist()
        for r in [q for q in (0, 2, WINDOW - 1) if not o_ann[q]]:
            assert self.cl.debugCounters(W0 + r)[0] == self.sim.updatesInProgress(r), "receiver %d" % (W0 + r)

    def gets(self):
        return np.array([_gets(r) for r in range(R)]) if self.bitmap else np.ones(R, bool)

    def check_in_band(self, res):
        """after the L batch: nothing emitted, every receiver that got the cells has N_WIDE subjects in progress"""
        assert (res.proposal_len == 0).all() and (res.announced == 0).all()
        gets = self.gets()
        for r in list(range(0, R, 97)) + [R - 1]:
            assert self.cl.debugCounters(r)[0] == (N_WIDE if gets[r] else 0), "receiver %d" % r

    def check_announced(self, res):
        """after the H batch: every receiver that got the cells announces all N_WIDE subjects"""
        gets = self.gets()
        np.testing.assert_array_equal(res.proposal_len, np.where(gets, N_WIDE, 0))
        np.testing.assert_array_equal(res.announced, gets.astype(np.uint8))
        assert (res.proposal_hash[gets] == np.uint64(self.want[0])).all()
        assert (res.proposal_hash2[gets] == np.uint64(self.want[1])).all()
        r = int(np.nonzero(gets)[0][-1])
        assert sorted(self.cl.getProposal(r, cap=N_WIDE + 8)) == self.d["subjects"].tolist()


def test_wide_batch_default_grid(world):
    """(a) 70,000 fresh subjects reach L in one batch (the batch-wide fresh totals), then all of them reach H"""
    _default_grid(world)


def test_wide_batch_in_one_chunk(world):
    """(b) a duplicate-heavy batch first makes the host's estimate 1 subject, so the wide batches run in ONE subject chunk: the
    chunk record sums 70,000 fresh L-crossings, and the carried subjects of the H batch sum 70,000 H-crossings in every
    receiver's partials"""
    _in_one_chunk(world)


@pytest.mark.parametrize("one_chunk", [False, True])
def test_wide_sequence_prefix(world, one_chunk):
    """(c) one sequence call: the prefix moves 70,000 subjects into the band, the last batch moves them to H (one pass)"""
    _sequence_prefix(world, one_chunk)


def test_wide_batch_bitmap_delivery(world):
    """(d) per-receiver delivery bitmaps (the generic kernel) in one subject chunk: one receiver in five gets no cell"""
    _bitmap_delivery(world)


@pytest.mark.parametrize("case", ["default", "one-chunk"])
def test_wide_batches_at_fourteen_rings(orc, case):
    """(a) and (b) at K = 14, where the rows hold a hi byte per receiver"""
    d = _world(orc, 14)
    {"default": _default_grid, "one-chunk": _in_one_chunk}[case](d)


def _default_grid(world):
    c = Case(world)
    c.check_in_band(c.batch(world["low"]))
    c.check_announced(c.batch(world["high"]))


def _in_one_chunk(world):
    c = Case(world)
    c.batch(world["dup"], oracle=False)                             # (uniform delivery, seen by the handle only)
    res = c.batch(world["low"])
    assert c.cl.debugGrid()[0] == 1
    c.check_in_band(res)
    c.batch(world["dup"], oracle=False)                             # (uniform delivery, seen by the handle only)
    res = c.batch(world["high"])
    assert c.cl.debugGrid()[0] == 1
    c.check_announced(res)


def _sequence_prefix(world, one_chunk):
    rb = world["rb"]
    c = Case(world)
    if one_chunk:
        c.batch(world["dup"], oracle=False)                             # (uniform delivery, seen by the handle only)
    lo, hi = world["low"], world["high"]
    src, dst, ring, status = (np.concatenate([a, b]) for a, b in zip(lo, hi))
    off = np.array([0, len(lo[1]), len(dst)], np.int64)
    res, ain = c.cl.handleBatches(world["cfg"], src, dst, ring, status, off)
    assert c.cl.sequenceStats() == (1, 0), c.cl.sequenceRefusal()
    if one_chunk:
        assert c.cl.debugGrid()[0] == 1
    np.testing.assert_array_equal(ain, np.full(R, 1, np.int32))
    c.check_announced(res)
    # the oracle handles the two batches one by one
    for b in range(2):
        sl = slice(int(off[b]), int(off[b + 1]))
        o_len, o_ann, o_ids, o_off = c.sim.apply_batch(src[sl], dst[sl], ring[sl], status[sl],
                                                       np.full(sl.stop - sl.start, world["cfg"], np.int64), threads=8)
        assert (o_len == 0).all() if b == 0 else (o_len == N_WIDE).all()
    c.compare(res, o_len, o_ann, o_ids, o_off)
    assert rb.proposal_fingerprint(o_ids[o_off[0]: o_off[1]]) == c.want


def _bitmap_delivery(world):
    c = Case(world, bitmap=True)
    c.batch(world["dup"], oracle=False)                             # (uniform delivery, seen by the handle only)
    res = c.batch(world["low"])
    assert c.cl.lastPath()[0] == 3 and c.cl.debugGrid()[0] == 1
    c.check_in_band(res)
    c.batch(world["dup"], oracle=False)                             # (uniform delivery, seen by the handle only)
    res = c.batch(world["high"])
    assert c.cl.lastPath()[0] == 3 and c.cl.debugGrid()[0] == 1
    c.check_announced(res)
