"""The bucketed detector's packed state rows vs the oracle.

A bucketed row keeps rings 0..7 in a byte plane and rings 8.., bit 14 and bit 15 in a hi plane of 4 bits per receiver when
K <= 10 (two receivers share a byte) and 8 bits when K > 10.  These tests aim at what that layout can get wrong: neighbouring
receivers whose hi lanes share a byte but hold different words, the widening of the hi plane from K = 10 to K = 11, and the
places that write single lanes (the generic kernel's per-receiver stores, the bit-15 marks).  Every receiver of a window that
crosses a 1024-receiver tile edge is compared with the oracle."""
import numpy as np
import pytest

from helpers import OracleWorld, compare_batch, random_batch

pytestmark = pytest.mark.gpu
DOWN = 1
N = 1100                                   # two tiles of 1024 receivers
WINDOW = range(1016, 1032)                 # across the tile edge: odd / even pairs on both sides
KHL = [(10, 9, 4), (11, 9, 4), (14, 12, 5)]


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


def _worlds(orc, rb, Kx, Hx, Lx):
    w = OracleWorld(orc, N, Kx)
    v = rb.MembershipView.from_packed(Kx, *w.member_packed())
    sim = orc.ClusterSim(w.view, Kx, Hx, Lx, N)
    cl = rb.VirtualCluster(v, Hx, Lx, kernel="bucketed")
    return w, v, sim, cl


def _check_window(cl, sim, o_ann):
    """the masks and updatesInProgress of every live receiver of the window (announced receivers' state is dead until clear())"""
    checked = 0
    for r in WINDOW:
        if o_ann[r]:
            continue
        for subj, m in cl.debugMasks(r).items():
            assert sim.reportMask(r, int(subj)) == m, "mask of subject %d at receiver %d" % (subj, r)
        assert cl.debugCounters(r)[0] == sim.updatesInProgress(r), "receiver %d" % r
        checked += 1
    return checked


@pytest.mark.parametrize("Kx,Hx,Lx", KHL)
def test_even_and_odd_receivers_get_different_cells(orc, rb, Kx, Hx, Lx):
    """per-receiver bitmaps (generic kernel): even receivers get the even cells, odd receivers the odd ones, so the hi lanes
    that share a byte diverge; state is carried from batch to batch"""
    w, v, sim, cl = _worlds(orc, rb, Kx, Hx, Lx)
    rng = np.random.default_rng(Kx)
    words = (N + 31) // 32
    checked = 0
    for _ in range(4):
        src, dst, ring, status = random_batch(rng, N, Kx, int(rng.integers(3, 8)), int(rng.integers(20, 70)), N)
        bitmap = np.where((np.arange(len(dst)) % 2 == 0)[:, None], np.uint32(0x55555555), np.uint32(0xAAAAAAAA))
        bitmap = np.repeat(bitmap, words, axis=1).astype(np.uint32)
        bitmap[rng.random(len(dst)) < 0.2] = 0xFFFFFFFF                 # a few cells reach everyone
        _, o_ann = compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), bitmap=bitmap)
        checked += _check_window(cl, sim, o_ann)
    assert checked > 0


@pytest.mark.parametrize("Kx,Hx,Lx", KHL)
def test_alternate_receivers_blocked_then_carried(orc, rb, Kx, Hx, Lx):
    """uniform delivery (SWAR kernel) with every other receiver blocked, then batches that reach everyone: the carried
    words of neighbouring receivers differ, and the per-receiver fallback unpacks and packs them again"""
    w, v, sim, cl = _worlds(orc, rb, Kx, Hx, Lx)
    rng = np.random.default_rng(50 + Kx)
    odd = (np.arange(N) % 2).astype(np.uint8)
    checked = 0
    for blocked in (odd, None, 1 - odd, None):
        src, dst, ring, status = random_batch(rng, N, Kx, int(rng.integers(3, 8)), int(rng.integers(10, 50)), N)
        _, o_ann = compare_batch(rb, w, sim, cl, None, (src, dst, ring, status), blocked=blocked)
        checked += _check_window(cl, sim, o_ann)
    assert checked > 0


@pytest.mark.parametrize("Kx,Hx,Lx", KHL)
def test_bit15_marks_on_alternate_receivers(orc, rb, Kx, Hx, Lx):
    """A leaves in an explicit proposal, then X and one of its observers enter the unstable band and stay there: the
    receivers announce only the explicit part {A}, which is kept as bit-15 marks.  Odd receivers are blocked, so the marks
    land on every other receiver; the odd ones carry on with the next batch and their words must be untouched."""
    rng = np.random.default_rng(700 + Kx)
    odd = (np.arange(N) % 2).astype(np.uint8)
    hits = 0
    for trial in range(8):
        w, v, sim, cl = _worlds(orc, rb, Kx, Hx, Lx)
        obs, _ = v.tables()
        x = int(rng.integers(0, N))
        xo = obs[x].tolist()
        o1 = xo[int(rng.integers(0, Kx))]
        rings_x = [k for k in range(Kx) if xo[k] != o1][: Hx - 1]        # X ends one short of H, none of it via o1
        if len(rings_x) < Lx or o1 == x:
            continue
        a = int(rng.choice([i for i in range(N) if i not in (x, o1) and i not in xo and i not in obs[o1].tolist()]))
        first = [(a, int(k)) for k in rng.permutation(Kx)[:Hx]]
        late = [(x, k) for k in rings_x] + [(o1, int(k)) for k in rng.permutation(Kx)[: int(rng.integers(Lx, Hx))]]
        rng.shuffle(late)
        cells = first + late
        dst = np.array([c[0] for c in cells], np.int32)
        ring = np.array([c[1] for c in cells], np.uint8)
        o_len, o_ann = compare_batch(rb, w, sim, cl, None, (np.zeros(len(cells), np.int32), dst, ring, np.full(len(cells), DOWN, np.uint8)),
                                     blocked=odd)
        if (o_len[odd == 0] == 1).all():
            hits += 1
            for r in WINDOW[::2]:
                assert cl.getProposal(r) == [a], "receiver %d" % r
        _check_window(cl, sim, o_ann)
        # the odd receivers carry on; the even ones announced and ignore it
        src2, dst2, ring2, st2 = random_batch(rng, N, Kx, 3, 25, N)
        _, o_ann = compare_batch(rb, w, sim, cl, None, (src2, dst2, ring2, st2))
        assert _check_window(cl, sim, o_ann) > 0
    assert hits > 0
