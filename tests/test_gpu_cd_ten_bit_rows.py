"""The bucketed detector's ring-bit-only rows and its two mark planes vs the oracle.

At K <= 10 a bucketed row keeps rings 0..7 in a byte plane and rings 8, 9 in a hi plane of 2 bits per receiver: four receivers
share a hi byte, and the generic kernel stores the hi lanes of 16 receivers as one word.  The emitted mark (bit 15) and the
invalidation pass's transient mark (bit 14) live in planes of one bit per (slot, receiver) beside the rows.  These tests aim at
what that layout can get wrong: neighbouring receivers whose hi lanes share a byte or a word but hold different words, stale
emit marks after clear() reuses the slots, a transient mark that is not cleared before the next batch, and the sequence
kernels' loads of their observers' rows.  Receivers of a window that crosses a 1024-receiver tile edge are compared with the
oracle."""
import numpy as np
import pytest

from helpers import OracleWorld, compare_batch, fingerprints_from_oracle, random_batch

pytestmark = pytest.mark.gpu
DOWN = 1
N = 1100                                   # two tiles of 1024 receivers
WINDOW = range(1008, 1040)                 # across the tile edge: two hi words on each side
KHL = [(10, 9, 4), (11, 9, 4)]


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


def _worlds(orc, rb, Kx, Hx, Lx, n=N):
    w = OracleWorld(orc, n, Kx)
    v = rb.MembershipView.from_packed(Kx, *w.member_packed())
    sim = orc.ClusterSim(w.view, Kx, Hx, Lx, n)
    cl = rb.VirtualCluster(v, Hx, Lx, kernel="bucketed")
    return w, v, sim, cl


def _check_window(cl, sim, o_ann, window=WINDOW):
    """the masks and updatesInProgress of every live receiver of the window (announced receivers' state is dead until clear())"""
    checked = 0
    for r in window:
        if o_ann[r]:
            continue
        for subj, m in cl.debugMasks(r).items():
            assert sim.reportMask(r, int(subj)) == m, "mask of subject %d at receiver %d" % (subj, r)
        assert cl.debugCounters(r)[0] == sim.updatesInProgress(r), "receiver %d" % r
        checked += 1
    return checked


def _pool_batch(rng, pool, Kx, n_cells):
    """cells about a small fixed pool of subjects, so that most of them are carried from batch to batch"""
    dst = rng.choice(pool, size=n_cells).astype(np.int32)
    ring = rng.integers(0, Kx, size=n_cells).astype(np.uint8)
    src = rng.integers(0, N, size=n_cells).astype(np.int32)
    return src, dst, ring, np.full(n_cells, DOWN, np.uint8)


@pytest.mark.parametrize("pattern", ["blocked4", "blocked3", "bitmap4"])
@pytest.mark.parametrize("Kx,Hx,Lx", KHL)
def test_receivers_of_a_hi_byte_and_word_diverge(orc, rb, Kx, Hx, Lx, pattern):
    """blocked receivers with periods 4 and 3 (SWAR kernel) and per-receiver bitmaps with period 4 (generic kernel, the 16-lane
    warp store): the phase moves from batch to batch and state is carried, so the four receivers of a hi byte and the sixteen of
    a hi word end up holding different words in every position"""
    w, v, sim, cl = _worlds(orc, rb, Kx, Hx, Lx)
    rng = np.random.default_rng(Kx * 10 + len(pattern))
    pool = rng.choice(N, size=24, replace=False)
    words = (N + 31) // 32
    checked = 0
    for b in range(6):
        src, dst, ring, status = _pool_batch(rng, pool, Kx, int(rng.integers(20, 60)))
        kw = {}
        if pattern.startswith("blocked"):
            period = int(pattern[-1])
            kw["blocked"] = ((np.arange(N) % period) == (b % period)).astype(np.uint8)
        else:
            lane = np.arange(32)
            phase = (np.arange(len(dst)) + b) % 4
            bits = ((lane[None, :] % 4) == phase[:, None]) | ((lane[None, :] % 4) == ((phase[:, None] + b) % 4))
            word = (bits.astype(np.uint64) << lane[None, :].astype(np.uint64)).sum(axis=1).astype(np.uint32)
            bitmap = np.repeat(word[:, None], words, axis=1).astype(np.uint32)
            bitmap[rng.random(len(dst)) < 0.1] = 0xFFFFFFFF                  # a few cells reach everyone
            kw["bitmap"] = bitmap
        _, o_ann = compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), **kw)
        if pattern == "bitmap4":
            assert cl.lastPath()[0] == 3
        checked += _check_window(cl, sim, o_ann)
    assert checked > 0


def _explicit_only(rng, obs, n, Kx, Hx, Lx):
    """A leaves in an explicit proposal, then X and one of its observers enter the unstable band and stay there: the receivers
    announce only the explicit part {A}.  None if the draw does not fit."""
    x = int(rng.integers(0, n))
    xo = obs[x].tolist()
    o1 = xo[int(rng.integers(0, Kx))]
    rings_x = [k for k in range(Kx) if xo[k] != o1][: Hx - 1]
    if len(rings_x) < Lx or o1 == x:
        return None
    a = int(rng.choice([i for i in range(n) if i not in (x, o1) and i not in xo and i not in obs[o1].tolist()]))
    first = [(a, int(k)) for k in rng.permutation(Kx)[:Hx]]
    late = [(x, k) for k in rings_x] + [(o1, int(k)) for k in rng.permutation(Kx)[: int(rng.integers(Lx, Hx))]]
    rng.shuffle(late)
    cells = first + late
    dst = np.array([c[0] for c in cells], np.int32)
    ring = np.array([c[1] for c in cells], np.uint8)
    return a, (np.zeros(len(cells), np.int32), dst, ring, np.full(len(cells), DOWN, np.uint8))


@pytest.mark.parametrize("Kx,Hx,Lx", KHL)
def test_emit_marks_survive_new_slots_and_do_not_leak_past_clear(orc, rb, Kx, Hx, Lx):
    """Explicit-only announcements land on the receivers r % 4 == k (the others are blocked).  Later batches assign new slots
    while the other receivers go on, and every marked receiver must still list exactly {A}.  Then clear() and a second epoch
    reuses the slots with the marks on other receivers: no mark of the first epoch may leak into any getProposal."""
    rng = np.random.default_rng(900 + Kx)
    w, v, sim, cl = _worlds(orc, rb, Kx, Hx, Lx)
    obs, _ = v.tables()
    hits = 0
    for epoch, k in enumerate([0, 1, 2, 3, 2, 0]):
        if epoch:
            cl.clear(); sim.reset()
        drawn = None
        while drawn is None:
            drawn = _explicit_only(rng, obs, N, Kx, Hx, Lx)
        a, cells = drawn
        marked = (np.arange(N) % 4) == k
        o_len, o_ann = compare_batch(rb, w, sim, cl, None, cells, blocked=(~marked).astype(np.uint8))
        if not (o_len[marked] == 1).all():
            continue
        hits += 1
        for _ in range(2):                                              # new slots while the other receivers carry on
            src2, dst2, ring2, st2 = random_batch(rng, N, Kx, 6, 40, N)
            _, o_ann = compare_batch(rb, w, sim, cl, None, (src2, dst2, ring2, st2))
            _check_window(cl, sim, o_ann)
        for r in WINDOW:
            if marked[r]:
                assert cl.getProposal(r) == [a], "receiver %d, epoch %d" % (r, epoch)
    assert hits >= 2


def test_transient_marks_of_the_invalidation_pass_are_cleared(orc, rb):
    """Subjects reported in an earlier batch sit in the band and are not touched by the next one; in that next batch some
    receivers emit early and then see subjects stay in the band (MIXED, the interval analysis), and the invalidation pass raises
    carried subjects.  The transient marks it leaves must be gone before the next batch: every trial reuses the slots of the
    one before (clear()), where a stale mark would turn a pending subject into a raised one."""
    n, Kx = 40, 10
    rng = np.random.default_rng(4242)
    seen = []
    Hh, Ll = 8, 3
    w, v, sim, cl = _worlds(orc, rb, Kx, Hh, Ll, n=n)
    obs, _ = v.tables()
    for trial in range(40):
        cl.clear(); sim.reset()
        s = int(rng.integers(0, n))
        o = list(dict.fromkeys(obs[s].tolist()))
        rng.shuffle(o)
        early = o[: int(rng.integers(1, 4))]
        carried = [x for x in o[len(early):]][: int(rng.integers(1, 5))]   # into the band one batch ahead
        pend = int(rng.choice([i for i in range(n) if i != s and i not in o]))
        cells = [(c, int(k)) for c in carried for k in rng.permutation(Kx)[: int(rng.integers(Ll, Hh))]]
        cells += [(pend, int(k)) for k in rng.permutation(Kx)[: int(rng.integers(Hh, Kx + 1))]] if trial % 2 else []
        rng.shuffle(cells)
        b1 = (np.zeros(len(cells), np.int32), np.array([c[0] for c in cells], np.int32),
              np.array([c[1] for c in cells], np.uint8), np.full(len(cells), DOWN, np.uint8))
        # (on odd trials `pend` reaches H in this batch: pending wherever a carried subject is still in the band)
        compare_batch(rb, w, sim, cl, None, b1, blocked=(np.arange(n) % 3 == 0).astype(np.uint8) if trial % 3 == 0 else None)
        cells = []
        for e in early:
            cells += [(e, int(k)) for k in rng.permutation(Kx)[: int(rng.integers(Hh, Kx + 1))]]
        late = [(s, int(k)) for k in rng.permutation(Kx)[: int(rng.integers(Ll, Hh))]]
        rng.shuffle(late)
        cells += late
        b2 = (np.zeros(len(cells), np.int32), np.array([c[0] for c in cells], np.int32),
              np.array([c[1] for c in cells], np.uint8), np.full(len(cells), DOWN, np.uint8))
        compare_batch(rb, w, sim, cl, None, b2)
        n_mixed, n_pairs = cl.debugStats()[:2]
        seen.append((n_mixed, n_pairs))
        src3, dst3, ring3, st3 = random_batch(rng, n, Kx, 4, 30, n)
        compare_batch(rb, w, sim, cl, None, (src3, dst3, ring3, st3))
    both = [x for x in seen if x[0] > 0 and x[1] > 0]
    assert len(both) >= 2, seen                                          # MIXED batches with inval pairs, more than once


@pytest.mark.parametrize("Kx,Hx,Lx", KHL)
def test_sequence_kernels_read_their_observers_rows(orc, rb, Kx, Hx, Lx):
    """a sequence of batches in one call (C4 shape) about subjects whose observers are subjects too, with state carried from
    call to call: the sequence kernels load the observers' rows in the ring-bit format"""
    w, v, sim, cl = _worlds(orc, rb, Kx, Hx, Lx)
    obs, _ = v.tables()
    rng = np.random.default_rng(31 + Kx)
    cfg = w.view.getCurrentConfigurationId()
    served = 0
    for call in range(3):
        subj = [int(x) for x in rng.choice(N, size=6, replace=False)]
        subj += [int(obs[s][int(rng.integers(0, Kx))]) for s in subj[:3]]   # dictionary observers
        batches = [_pool_batch(rng, np.asarray(subj), Kx, int(rng.integers(4, 14))) for _ in range(3)]
        ln, h1, h2 = np.zeros(N, np.int32), np.zeros(N, np.uint64), np.zeros(N, np.uint64)
        ain = np.full(N, -1, np.int32)
        for b, (src, dst, ring, status) in enumerate(batches):
            o_len, o_ann, o_ids, o_off = sim.apply_batch(src, dst, ring, status, np.full(len(dst), cfg, np.int64), threads=4)
            e1, e2 = fingerprints_from_oracle(rb, o_len, o_ids, o_off)
            now = o_len > 0
            ain[now] = b; ln[now] = o_len[now]; h1[now] = e1[now]; h2[now] = e2[now]
        src, dst, ring, status = (np.concatenate(x) for x in zip(*batches))
        off = np.concatenate([[0], np.cumsum([len(x[1]) for x in batches])]).astype(np.int64)
        res, g_ain = cl.handleBatches(cfg, src, dst, ring, status, off)
        np.testing.assert_array_equal(g_ain, ain)
        np.testing.assert_array_equal(res.proposal_len, ln)
        np.testing.assert_array_equal(res.proposal_hash, h1)
        np.testing.assert_array_equal(res.proposal_hash2, h2)
        np.testing.assert_array_equal(res.announced, o_ann)
        _check_window(cl, sim, o_ann)
        served = cl.sequenceStats()[0]
    assert served > 0
