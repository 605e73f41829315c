"""The subject-bucketed cut detector under every grid shape, against one recording of the literal oracle.

The host sizes the apply kernels' grid (tiles x subject chunks) from an ESTIMATE of the batch's subject count and k_prepare's
grid from the cell count; the kernels split the real count on the device.  Small inputs always take the same shape, so here
one seeded mid-scale stream is recorded once per delivery mode through the oracle and replayed on a fresh handle per shape:
forced chunk counts (RAPID_B200_CHUNKS) that put 31, 32, 33, 64 and 65 subjects in a chunk, more chunks than subjects, forced
k_prepare grids (RAPID_B200_PREP_GRID), and the default heuristic fed batches whose cells-per-subject ratio swings by 10x either
way.  Every forced shape is checked to have been taken (VirtualCluster.debugGrid).

The world is built at every ring count whose row format differs: K = 3, K = 8 (the last whose hi plane is always empty), K = 10
(the last with two hi bits per receiver), K = 11 (the first with a hi byte per receiver) and K = 14 (RAPID_MAX_K), each with two
(H, L) pairs, one of them at an edge (H = K, or H close to L).  Each pair keeps a non-empty unstable band (L < H), so the
uniform and permuted cases can be checked to have taken the interval analysis, and every sequence-mode case to have served a call
in one pass (the SEQ kernels under every shape)."""
import numpy as np
import pytest

from helpers import OracleWorld, fingerprints_from_oracle
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu
N, NJ = 4000, 6
R, BEGIN = 2901, 555                  # three tiles of 1024 receivers, the last one partial; R is not a multiple of 8
SAMPLE = [0, 7, 8, 1023, 1024, 1500, 2047, 2048, 2900]
# distinct subjects per batch: with 5 chunks 31 and 32 per chunk (batches 0 and 3), with 3 chunks 33 (batch 2), with 2 chunks
# 64 and 65 (batches 1 and 4); cells per subject swing between ~1 and ~K so the default estimate is off by 10x both ways
# (batches 6 and 7: 150 subjects, the same in both)
COUNTS = [155, 128, 99, 160, 130, 262, 150, 150]
SHAPE = ["mid", "one", "many", "many", "one", "mid", "many", "mid"]
# sequence modes: three handleBatches calls.  Both handles are cleared before batch 6 (the detector's clear(), the oracle's
# reset()), and the third call's prefix keeps its subjects in the band until its last batch, so that call is served in one pass.
CALLS = [(0, 3), (3, 6), (6, 8)]
RESET = 6
HEAVY = 3000                          # batch 5: one subject's cells spread over every k_prepare block (bins past 64 cells)


def _stream(obs, K, Hh, Ll, seed):
    """Subjects are carried from batch to batch (about half of every batch); each one is pushed below L, into the band or to
    all K rings.  Batch 3 first completes every subject still in the band, then brings new ones into it (a receiver that got
    everything emits mid-batch and then sees subjects enter the band: the interval analysis); batch 5 completes them at its end.
    Then the state is cleared: batch 6 pushes fresh subjects below L or into the band (never to H, with duplicates), batch 7
    brings every one of them to all K rings."""
    rng = np.random.default_rng(seed)
    n_total = N + NJ
    rings_of = {}
    batches = []
    for b, (ns, shape) in enumerate(zip(COUNTS, SHAPE)):
        if b >= RESET:
            batches.append(_after_reset(obs, K, Hh, Ll, rng, rings_of, b, ns, shape))
            continue
        band = [s for s, x in rings_of.items() if Ll <= len(x) < Hh]
        drain = band if b in (3, 5) else []
        assert len(drain) <= ns - 20
        open_ = [s for s, x in rings_of.items() if len(x) < K and s not in drain]
        n_car = min(len(open_), max(0, ns // 2 - len(drain)))
        car = [int(x) for x in rng.choice(np.asarray(open_), size=n_car, replace=False)] if n_car else []
        heavy = []
        pool = np.setdiff1d(np.arange(n_total), np.asarray(list(rings_of), np.int64))
        if b == 5:
            heavy = [int(rng.choice(pool))]
            pool = pool[pool != heavy[0]]
        fresh = [int(x) for x in rng.choice(pool, size=ns - len(drain) - n_car - len(heavy), replace=False)]
        first, cells = [], []
        for s in drain:
            first += [(s, k) for k in range(K) if k not in rings_of[s]]
        for s in car + fresh:
            have = rings_of.get(s, set())
            missing = [k for k in range(K) if k not in have]
            if shape == "one":
                new = [int(rng.choice(missing))]
            else:
                target = [int(rng.integers(len(have) + 1, max(Ll, len(have) + 1) + 1)),      # below L or just into the band
                          int(rng.integers(max(Ll, len(have) + 1), max(Hh, len(have) + 1) + 1)), K][int(rng.integers(0, 3))]
                new = [int(k) for k in rng.choice(missing, size=min(len(missing), max(1, target - len(have))), replace=False)]
            dups = list(rng.choice(list(have | set(new)), size=int(rng.integers(2, 5)))) if shape == "many" else []
            cells += [(s, int(k)) for k in new + dups]
        cells = [cells[i] for i in rng.permutation(len(cells))]
        cells = first + cells if b == 3 else cells + first
        if b == 5:
            pos = set(rng.choice(len(cells) + HEAVY, size=HEAVY, replace=False).tolist())
            it, hv = iter(cells), iter(rng.integers(0, K, size=HEAVY).tolist())
            cells = [(heavy[0], next(hv)) if i in pos else next(it) for i in range(len(cells) + HEAVY)]
        for s, k in cells:
            rings_of.setdefault(s, set()).add(k)
        dst = np.array([c[0] for c in cells], np.int32)
        ring = np.array([c[1] for c in cells], np.uint8)
        src = obs[dst, ring].astype(np.int32)
        status = np.where(dst < N, W.DOWN, W.UP).astype(np.uint8)
        assert len(np.unique(dst)) == ns
        batches.append((src, dst, ring, status))
    return batches


def _after_reset(obs, K, Hh, Ll, rng, rings_of, b, ns, shape):
    """batch 6 (state cleared before it) or 7 of the stream"""
    if b == RESET:
        # no subject observes another: no invalidation pass at the end of batch 6 can report a ring implicitly and carry a subject
        # to H inside the prefix
        rings_of.clear()
        subjects, watchers = [], set()                         # watchers: the observers of the subjects taken
        for x in rng.permutation(N + NJ).tolist():
            if len(subjects) == ns:
                break
            if x not in watchers and not set(subjects).intersection(obs[x].tolist()):
                subjects.append(x)
                watchers.update(obs[x].tolist())
    else:
        subjects = list(rings_of)
    cells = []
    for s in subjects:
        have = rings_of.get(s, set())
        missing = [k for k in range(K) if k not in have]
        if b == RESET:                                             # into the band, or below L (when L > 1)
            lo, hi = (Ll, Hh - 1) if Ll == 1 or rng.random() < 0.7 else (1, Ll - 1)
            new = [int(k) for k in rng.choice(missing, size=int(rng.integers(lo, hi + 1)), replace=False)]
        else:                                                      # every missing ring: the band's subjects cross H here
            new = missing
        dups = list(rng.choice(list(have | set(new)), size=int(rng.integers(2, 5)))) if shape == "many" else []
        cells += [(s, int(k)) for k in new + dups]
    cells = [cells[i] for i in rng.permutation(len(cells))]
    for s, k in cells:
        rings_of.setdefault(s, set()).add(k)
    if b == RESET:
        assert max(len(x) for x in rings_of.values()) < Hh and any(len(x) >= Ll for x in rings_of.values())
    else:
        assert all(len(x) == K for x in rings_of.values())
    dst = np.array([c[0] for c in cells], np.int32)
    ring = np.array([c[1] for c in cells], np.uint8)
    src = obs[dst, ring].astype(np.int32)
    status = np.where(dst < N, W.DOWN, W.UP).astype(np.uint8)
    assert len(np.unique(dst)) == ns
    return src, dst, ring, status


def _delivery(mode, b, rng):
    """blocked receivers, bitmaps and permutation seeds of batch b"""
    kw = {}
    if b in (1, 3):
        kw["blocked"] = (rng.random(R) < (0.1 if b == 1 else 0.3)).astype(np.uint8)
    if b == 7:
        kw["blocked"] = (rng.random(R) < 0.2).astype(np.uint8)
    if b in (2, 4):
        bl = np.zeros(R, np.uint8)
        bl[(np.arange(R) % 1024) < 9] = 1                          # every tile's first receivers: the memo's sample moves
        if b == 2:
            bl[1024: 2048] = 1                                    # a tile with no active receiver
        kw["blocked"] = bl
    if mode == "bitmap" or (mode == "mixed" and b == 0):
        kw["bitmap"] = None                                        # filled per batch (needs the cell count)
    if mode in ("permuted", "seq_permuted"):
        kw["perm_seed"] = 0x5EED0000 + 17 * b
    return kw


_RECORD = {}
_WORLD = {}


@pytest.fixture(scope="module", autouse=True)
def _free_worlds():
    """the views and the recordings live as long as this module's tests"""
    yield
    _WORLD.clear()
    _RECORD.clear()


def _world(orc, K):
    """the view at K rings, built once per K"""
    if K not in _WORLD:
        import rapid_b200 as rb
        w = OracleWorld(orc, N, K, n_joiners=NJ)
        v = rb.MembershipView.from_packed(K, *w.member_packed())
        v.registerJoiners(*w.joiner_endpoints())
        obs = np.concatenate([w.tables()[0], w.joiner_obs()]).astype(np.int32)
        _WORLD[K] = dict(rb=rb, w=w, v=v, K=K, obs=obs, cfg=w.view.getCurrentConfigurationId())
    return _WORLD[K]


def _masks(sim, r, subjects):
    return {s: m for s in subjects if (m := sim.reportMask(r, s))}


def _record(world, orc, Hh, Ll, mode):
    """the oracle over the whole stream, once per (K, H, L, mode): per batch (or per sequence call) every receiver's outputs"""
    K = world["K"]
    key = (K, Hh, Ll, mode)
    if key in _RECORD:
        return _RECORD[key]
    rb, w = world["rb"], world["w"]
    batches = _stream(world["obs"], K, Hh, Ll, seed=Hh * 100 + Ll if K == 10 else (K, Hh, Ll))
    rng = np.random.default_rng(4242)
    deliveries = []
    for b, (src, dst, ring, status) in enumerate(batches):
        kw = _delivery(mode, b, rng)
        if "bitmap" in kw:
            words = (R + 31) // 32
            bm = rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
            kw["bitmap"] = bm | rng.integers(0, 2**32, size=(len(dst), words), dtype=np.uint64).astype(np.uint32)
        deliveries.append(kw)
    if mode.startswith("seq"):
        # one delivery per call: the blocked receivers of the call's second batch, batch b permuted with seed + (b - first)
        for b0, b1 in CALLS:
            base = deliveries[b0]
            blocked = deliveries[b0 + 1].get("blocked")
            for b in range(b0, b1):
                d = {} if blocked is None else {"blocked": blocked}
                if "perm_seed" in base:
                    d["perm_seed"] = base["perm_seed"] + (b - b0)
                deliveries[b] = d
    sim = orc.ClusterSim(w.view, K, Hh, Ll, R, receiver_base=BEGIN)
    cfg = world["cfg"]
    subjects = set()
    steps = []
    seq = mode.startswith("seq")
    groups = CALLS if seq else [(b, b + 1) for b in range(len(batches))]
    for b0, b1 in groups:
        if b0 == RESET:
            sim.reset()
            subjects = set()
        ln = np.zeros(R, np.int32); h1 = np.zeros(R, np.uint64); h2 = np.zeros(R, np.uint64)
        ain = np.full(R, -1, np.int32); ids = {}
        for b in range(b0, b1):
            src, dst, ring, status = batches[b]
            subjects |= set(dst.tolist())
            o_len, o_ann, o_ids, o_off = sim.apply_batch(src, dst, ring, status, np.full(len(dst), cfg, np.int64), threads=8,
                                                         **deliveries[b])
            e1, e2 = fingerprints_from_oracle(rb, o_len, o_ids, o_off)
            now = o_len > 0
            assert (ain[now] == -1).all()
            ain[now] = b - b0; ln[now] = o_len[now]; h1[now] = e1[now]; h2[now] = e2[now]
            for r in np.nonzero(now)[0][:: 97]:
                ids[int(r)] = o_ids[o_off[r]: o_off[r + 1]].tolist()
        masks = {r: (_masks(sim, r, sorted(subjects)), sim.updatesInProgress(r)) for r in SAMPLE if not o_ann[r]}
        steps.append(dict(range=(b0, b1), reset=b0 == RESET, len=ln, h1=h1, h2=h2, ann=o_ann.copy(), ain=ain, ids=ids, masks=masks))
    _RECORD[key] = (batches, deliveries, steps)
    return _RECORD[key]


SHAPES = [
    ("default", {}),
    ("chunks-1", {"RAPID_B200_CHUNKS": "1"}),
    ("chunks-2", {"RAPID_B200_CHUNKS": "2"}),
    ("chunks-3", {"RAPID_B200_CHUNKS": "3"}),
    ("chunks-5", {"RAPID_B200_CHUNKS": "5"}),
    ("chunks-over", {"RAPID_B200_CHUNKS": "100000"}),
    ("prep-1", {"RAPID_B200_PREP_GRID": "1"}),
    ("prep-3", {"RAPID_B200_PREP_GRID": "3"}),
    ("prep-max", {"RAPID_B200_PREP_GRID": "100000"}),
]
MODES = ["uniform", "permuted", "bitmap", "mixed", "seq_uniform", "seq_permuted"]


# (K, H, L): K = 3; K = 8, the last K whose hi plane is always empty; K = 10, the last with two hi bits per receiver; K = 11, the first
# with a hi byte per receiver; K = 14, the largest.  Every K with an edge pair: H = K, or a band one ring wide.
KHL = [(3, 3, 1), (3, 2, 1), (8, 7, 3), (8, 8, 2), (10, 9, 4), (10, 3, 1), (11, 10, 4), (11, 11, 4), (14, 13, 5), (14, 14, 6)]
ALL_SHAPES_AT = (10, 11, 14)          # K = 3 and 8 run a subset of the shapes
SUBSET = ("default", "chunks-1", "chunks-5", "chunks-over", "prep-1", "prep-max")
CASES = [(K, Hh, Ll, mode, shape, env) for K, Hh, Ll in KHL for mode in MODES for shape, env in SHAPES
         if K in ALL_SHAPES_AT or shape in SUBSET]


@pytest.mark.parametrize("K,Hh,Ll,mode,shape,env", CASES, ids=["%d-%d-%s-%s%s" % (h, l, m, s, "" if k == 10 else "-K%d" % k) for k, h, l, m, s, _ in CASES])
def test_every_grid_shape_matches_the_recording(orc, monkeypatch, K, Hh, Ll, mode, shape, env):
    world = _world(orc, K)
    rb = world["rb"]
    batches, deliveries, steps = _record(world, orc, Hh, Ll, mode)
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    cl = rb.VirtualCluster(world["v"], Hh, Ll, n_receivers=R, receiver_begin=BEGIN, kernel="bucketed")
    cfg = world["cfg"]
    over = []
    paths = set()
    mixed = 0
    for st in steps:
        b0, b1 = st["range"]
        if st["reset"]:
            cl.clear()
        if mode.startswith("seq"):
            src, dst, ring, status = (np.concatenate(x) for x in zip(*batches[b0:b1]))
            off = np.concatenate([[0], np.cumsum([len(batches[b][1]) for b in range(b0, b1)])]).astype(np.int64)
            kw = dict(deliveries[b0])
            res, ain = cl.handleBatches(cfg, src, dst, ring, status, off, **kw)
            np.testing.assert_array_equal(ain, st["ain"])
        else:
            res = cl.handleBatch(cfg, *batches[b0], **deliveries[b0])
            paths.add(cl.lastPath()[0])
        mixed += cl.debugStats()[0]
        np.testing.assert_array_equal(res.proposal_len, st["len"])
        np.testing.assert_array_equal(res.proposal_hash, st["h1"])
        np.testing.assert_array_equal(res.proposal_hash2, st["h2"])
        np.testing.assert_array_equal(res.announced, st["ann"])
        for r, ids in st["ids"].items():
            assert cl.getProposal(r) == ids, "receiver %d" % r
        for r, (m, npre) in st["masks"].items():
            assert {s: x for s, x in cl.debugMasks(r).items() if x} == m, "masks of receiver %d" % r
            assert cl.debugCounters(r)[0] == npre, "receiver %d" % r
        chunks, blocks = cl.debugGrid()
        subj = cl.debugStats()[2]
        if "RAPID_B200_CHUNKS" in env and shape != "chunks-over":
            assert chunks == int(env["RAPID_B200_CHUNKS"])
        if shape == "chunks-over":
            over.append(chunks > subj)
        if shape in ("prep-1", "prep-3"):
            assert blocks == int(env["RAPID_B200_PREP_GRID"])
        if shape == "prep-max":
            assert blocks > 3
    if shape == "chunks-over":
        assert any(over)                                           # some batch ran with empty chunks
    want_paths = {"uniform": {2}, "mixed": {3, 2}, "permuted": {4}, "bitmap": {3}}
    if mode in want_paths:
        assert paths == want_paths[mode]
    # the stream did what it was built for: on the uniform and permuted kernels (which count it) some receiver emitted
    # mid-batch and then saw subjects enter the band
    if mode in ("uniform", "permuted"):
        assert mixed > 0
    if mode.startswith("seq"):
        assert cl.sequenceStats()[0] >= 1, cl.sequenceRefusal()       # the third call, at least, was served in one pass
