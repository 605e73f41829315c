"""The fast-round tally of a detector's own votes (csrc/fast_paxos.cu: k_fp_tally, the kernel that decides every bench.py step)
against plainref.FastRound, field by field, on votes that conflict.

The votes come from the detector itself.  A handful of nodes crash and every receiver hears of them; the alerts about a few
extra crashed subjects reach only some receivers (per-receiver BITMAP delivery), so receivers announce different cuts.  A
receiver that gets only some of a subject's alerts is stuck in the unstable band and does not vote.  Each case checks that the
detector produced exactly the intended proposals before it compares the tally:
  - two interleaved proposals, the quorum reached mid-array, inside a later block of the kernel and not at a block edge
  - the same with the quorum never reached
  - stuck receivers interleaved with the voters
  - six extra subjects on random subsets: tens of distinct proposals, more than 16 in one block, with and without a winner
  - three calls: the first stays below the quorum, the second crosses it, the third changes nothing
The sharded tally (count-weighted sums, exact division, 12-bit-bucket refinement) runs the same cases on one GPU through a
one-rank NCCL communicator; it counts every vote of a call, so it is compared with the reference's totals.
The CPU test pins plainref.FastRound against the oracle's FastPaxosTally."""
import os

import numpy as np
import pytest

import plainref
from rapid_b200 import workloads as W

K, H, L = 10, 9, 4
BLOCK = 256                 # k_fp_tally gives every block a multiple of 256 receivers


# ---------------------------------------------------------------- the reference itself, against the oracle (CPU) ------------------
@pytest.mark.parametrize("seed", range(24))
def test_plain_fast_round_matches_oracle(orc, seed):
    rng = np.random.default_rng(300 + seed)
    N = int(rng.integers(4, 150))
    cap = N + 10
    nprop = int(rng.integers(1, 5))
    props = [sorted(rng.choice(1000, size=int(rng.integers(1, 5)), replace=False).tolist()) for _ in range(nprop)]
    weights = rng.dirichlet(np.ones(nprop) * 0.5)
    u = orc.Universe()
    stags = [u.add("s", s) for s in range(cap)]
    ptags = [[u.add("p", x) for x in p] for p in props]
    ofp = orc.FastPaxosTally(u, 5, N)
    ref = plainref.FastRound(N)
    for call in range(int(rng.integers(1, 5))):
        nv = int(rng.integers(0, 2 * N))
        senders = rng.integers(0, cap, size=nv)                  # repeated senders: only the first vote counts
        pid = rng.choice(nprop, size=nv, p=weights)
        for s, p in zip(senders, pid):
            ofp.handleFastRoundProposal(stags[s], 5, ptags[p])
        ref.call(senders, pid.tolist())
        assert ref.decided == ofp.decided() and ref.votes_received == ofp.votesReceived(), (seed, call)
        if ref.decided:
            assert ptags[ref.decision] == [int(x) for x in ofp.decision()]
            assert ref.count == ref.Q


def test_plain_fast_round_sharded_totals():
    ref = plainref.FastRound(8, sharded=True)                   # quorum 7
    ref.call([0, 1, 2, 3], ["a", "a", "b", "a"])
    assert not ref.decided and ref.votes_received == 4
    ref.call([4, 5, 6, 7, 1], ["a", "a", "a", "a", "b"])         # a reaches 7 at sender 7; the sender-1 repeat is ignored
    assert ref.decided and ref.decision == "a" and ref.count == 7 and ref.votes_received == 8
    ref.call([8], ["b"])
    assert ref.count == 7 and ref.votes_received == 8


# ---------------------------------------------------------------- detector-fed workloads -----------------------------------------
class World:
    def __init__(self, rb, n):
        hb, off, ports = W.packed_endpoints(0, n)
        self.n = n
        self.v = rb.MembershipView.from_packed(K, hb, off, ports)
        self.obs, _ = self.v.tables()
        self.ring0 = self.v.getRing(0)
        hi, lo = W.node_ids(0, n)
        self.cfg = self.v.getCurrentConfigurationId(hi, lo)


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.fixture(scope="module")
def worlds(rb):
    cache = {}

    def get(n):
        if n not in cache:
            cache[n] = World(rb, n)
        return cache[n]
    return get


def _row(hear):
    """delivery bitmap row: bit r of word r >> 5 set if receiver r gets the cell"""
    bits = np.zeros(((len(hear) + 31) // 32) * 32, bool)
    bits[: len(hear)] = hear
    return np.packbits(bits, bitorder="little").view(np.uint32)


def _pick_extras(rb, w, base, count, rng, bucket_of=None):
    """`count` more subjects that neither observe nor are observed by a crashed node, so each gets all K of its alerts;
    bucket_of: (h1 -> bucket, fingerprint to share it with): the first extra's cut must fall into that bucket"""
    failed = set(base.tolist())
    out = []
    while len(out) < count:
        x = int(rng.integers(w.n))
        row = set(w.obs[x].tolist())
        if x in failed or row & failed or any(x in set(w.obs[f].tolist()) for f in failed):
            continue
        if bucket_of is not None and not out:
            fn, want = bucket_of
            if fn(rb.proposal_fingerprint(np.sort(np.append(base, x)))[0]) != fn(want):
                continue
        failed.add(x)
        out.append(x)
    return np.asarray(out, np.int32)


class Votes:
    """one batch through the detector: who voted (receiver indices, in order), as which sender, for which proposal"""

    def __init__(self, w, res):
        self.who = np.nonzero(res.proposal_len > 0)[0]
        keyed = np.stack([res.proposal_hash[self.who], res.proposal_hash2[self.who], res.proposal_len[self.who].astype(np.uint64)], 1)
        uniq, pid = np.unique(keyed, axis=0, return_inverse=True)
        self.pid = pid.reshape(-1)
        self.props = [tuple(int(x) for x in row) for row in uniq]       # (hash, hash2, length)
        self.senders = w.ring0[self.who]

    def proposals(self):
        return [self.props[p] for p in self.pid.tolist()]


def run_batch(rb, w, cl, base, extras, hear, stuck, group=None):
    """crash `base` (heard by every receiver of `group`) and `extras` (extra j heard fully by receivers with hear[:, j], half of
    its alerts reach those with stuck[:, j]); check the detector's proposals against what that must give; return the votes"""
    n = w.n
    failed = np.sort(np.concatenate([base, extras])).astype(np.int32)
    cells = W.crash_cells(w.obs, failed, n)
    # the extras' alerts come first: a half-heard extra is then unstable before any crash reaches H, so it holds the whole cut
    # back (MultiNodeCutDetector releases a proposal whenever no subject is between L and H)
    first = np.argsort(~np.isin(cells["dst"], extras), kind="stable")
    cells = {k: a[first] for k, a in cells.items()}
    dst, ring = cells["dst"], cells["ring"]
    assert len(dst) == K * len(failed)
    group = np.ones(n, bool) if group is None else group
    rows = np.empty((len(dst), (n + 31) // 32), np.uint32)
    all_row = _row(group)
    rows[:] = all_row
    for j, x in enumerate(extras.tolist()):
        for k in range(K):
            sel = (dst == x) & (ring == k)
            rows[sel] = _row(group & (hear[:, j] | (stuck[:, j] & (k < K // 2))))
    bl = np.zeros(n, np.uint8)
    bl[failed] = 1
    blocked = W.blocked_by_receiver(bl, w.ring0, 0, n)
    res = cl.handleBatch(w.cfg, cells["src"], dst, ring, cells["status"], blocked=blocked, bitmap=rows)
    # what the detector must have announced: base + the extras heard in full, nothing while one is half heard
    assert not (hear & stuck).any()
    live = (blocked == 0) & group & ~stuck.any(1)
    code = (hear.astype(np.int64) << np.arange(len(extras))).sum(1)
    want_len = np.where(live, len(base) + hear.sum(1), 0)
    np.testing.assert_array_equal(res.proposal_len, want_len)
    for c in np.unique(code[live]).tolist():
        ids = np.sort(np.concatenate([base, extras[[(c >> j) & 1 == 1 for j in range(len(extras))]]]))
        h1, h2 = rb.proposal_fingerprint(ids)
        sel = live & (code == c)
        assert (res.proposal_hash[sel] == np.uint64(h1)).all() and (res.proposal_hash2[sel] == np.uint64(h2)).all()
    return Votes(w, res)


def check(t, ref, what):
    assert t.decided == ref.decided, what
    assert t.votes_received == ref.votes_received, what
    if ref.decided:
        assert (t.hash, t.hash2, t.length) == ref.decision, what
        assert t.count == ref.count, what


PATHS = ["in order", "sharded"]


class Arms:
    """the same detector outputs tallied by the in-order kernel, or by the sharded tally through a one-rank communicator, both
    through its sum buffer and forced onto its refinement path"""

    def __init__(self, rb, w, path, comm):
        if path == "in order":
            self.arms = [("in order", rb.FastPaxos(w.cfg, w.n), None, False, plainref.FastRound(w.n))]
        else:
            if comm is None:
                pytest.skip("the library could not load NCCL")
            self.arms = [("sharded", rb.FastPaxos(w.cfg, w.n), comm, False, plainref.FastRound(w.n, sharded=True)),
                         ("refined", rb.FastPaxos(w.cfg, w.n), comm, True, plainref.FastRound(w.n, sharded=True))]

    def tally(self, cl, votes):
        props = votes.proposals()
        for name, fp, comm, refine, ref in self.arms:
            if refine:
                os.environ["RAPID_B200_FORCE_REFINE"] = "1"
            try:
                t = fp.tallyCluster(cl, comm)
            finally:
                os.environ.pop("RAPID_B200_FORCE_REFINE", None)
            ref.call(votes.senders, props)
            check(t, ref, name)
        return self.arms[0][4]


@pytest.fixture(scope="module")
def comm(rb):
    """a one-rank NCCL communicator on device 0; None if the library cannot load NCCL"""
    try:
        import torch  # noqa: F401  (loads the libnccl.so.2 that torch ships, so the library's dlopen finds it)
        c = rb.NcclComm(0, 1, rb.NcclComm.unique_id(), 0)
    except (ImportError, rb.RapidError):
        yield None
        return
    yield c
    c.close()


def _interleaved_hear(w, rng, frac):
    """a fraction `frac` of the receivers hears the extra subject, interleaved at random"""
    return (rng.random(w.n) < frac)[:, None]


def _decided_at(votes, ref):
    """receiver index of the deciding vote"""
    return int(votes.who[ref.decided_at[1]])


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n", [20_000, 1_000_000])
def test_two_interleaved_proposals_quorum_mid_array(rb, worlds, comm, path, n):
    w = worlds(n)
    base = W.pick_smallest(n, 5, W.SEED + n)
    rng = np.random.default_rng(n)
    extras = _pick_extras(rb, w, base, 1, rng)
    none = np.zeros((n, 1), bool)
    for attempt in range(20):
        hear = _interleaved_hear(w, rng, 0.8)
        cl = rb.VirtualCluster(w.v, H, L)
        votes = run_batch(rb, w, cl, base, extras, hear, none)
        probe = plainref.FastRound(n)
        probe.call(votes.senders, votes.proposals())
        assert probe.decided and len(votes.props) == 2
        r = _decided_at(votes, probe)
        if r >= 4 * BLOCK and r % BLOCK not in (0, BLOCK - 1):     # inside a later block, not at its edge
            break
    else:
        pytest.fail("no draw put the deciding vote inside a block")
    ref = Arms(rb, w, path, comm).tally(cl, votes)
    assert ref.decided
    if path == "in order":
        assert ref.count == ref.Q and ref.votes_received < len(votes.who)     # votes after the decision are ignored


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n", [20_000, 100_000])
def test_two_interleaved_proposals_quorum_never_reached(rb, worlds, comm, path, n):
    w = worlds(n)
    base = W.pick_smallest(n, 4, W.SEED + 1)
    rng = np.random.default_rng(n + 1)
    extras = _pick_extras(rb, w, base, 1, rng)
    cl = rb.VirtualCluster(w.v, H, L)
    votes = run_batch(rb, w, cl, base, extras, _interleaved_hear(w, rng, 0.6), np.zeros((n, 1), bool))
    ref = Arms(rb, w, path, comm).tally(cl, votes)
    assert not ref.decided and ref.votes_received == len(votes.who) == n - 5


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n", [20_000, 100_000])
def test_stuck_receivers_interleaved_with_voters(rb, worlds, comm, path, n):
    """a tenth of the receivers get half the alerts of one extra subject: unstable, no vote; the rest split 85 : 5"""
    w = worlds(n)
    base = W.pick_smallest(n, 3, W.SEED + 2)
    rng = np.random.default_rng(n + 2)
    extras = _pick_extras(rb, w, base, 1, rng)
    u = rng.random(n)
    hear, stuck = (u < 0.85)[:, None], (u >= 0.9)[:, None]
    cl = rb.VirtualCluster(w.v, H, L)
    votes = run_batch(rb, w, cl, base, extras, hear, stuck)
    assert 0.08 * n < n - 4 - len(votes.who) < 0.12 * n
    ref = Arms(rb, w, path, comm).tally(cl, votes)
    assert ref.decided == (int((votes.pid == np.argmax(np.bincount(votes.pid))).sum()) >= ref.Q)


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n,dominant", [(20_000, False), (100_000, True), (20_000, True)])
def test_six_extra_subjects_many_proposals_per_block(rb, worlds, comm, path, n, dominant):
    """each receiver hears a random subset of six extra subjects: up to 64 proposals, more than 16 in one block (the overflow
    of the kernel's per-block table); with `dominant`, 80 % hear all six and that cut wins"""
    w = worlds(n)
    base = W.pick_smallest(n, 4, W.SEED + 3)
    rng = np.random.default_rng(n + 3 + dominant)
    extras = _pick_extras(rb, w, base, 6, rng)
    code = rng.integers(0, 64, size=n)
    if dominant:
        code = np.where(rng.random(n) < 0.8, 63, rng.integers(0, 63, size=n))
    hear = ((code[:, None] >> np.arange(6)) & 1).astype(bool)
    cl = rb.VirtualCluster(w.v, H, L)
    votes = run_batch(rb, w, cl, base, extras, hear, np.zeros((n, 6), bool))
    assert len(votes.props) > 40
    pairs = np.unique((votes.who // BLOCK) * len(votes.props) + votes.pid)        # distinct (block, proposal)
    assert np.bincount(pairs // len(votes.props)).max() > 16
    ref = Arms(rb, w, path, comm).tally(cl, votes)
    assert ref.decided == dominant


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n", [20_000, 100_000])
def test_count_carried_across_calls(rb, worlds, comm, path, n):
    """three batches reach three interleaved groups of receivers (45 %, 45 %, 10 %), one tally after each: the first stays
    below the quorum, the second crosses it mid-array while the proposals conflict, the third changes nothing"""
    w = worlds(n)
    base = W.pick_smallest(n, 4, W.SEED + 4)
    rng = np.random.default_rng(n + 4)
    extras = _pick_extras(rb, w, base, 1, rng)
    hear = _interleaved_hear(w, rng, 0.9)
    g = rng.random(n)
    groups = [g < 0.45, (g >= 0.45) & (g < 0.9), g >= 0.9]
    cl = rb.VirtualCluster(w.v, H, L)
    arms = Arms(rb, w, path, comm)
    seen = []
    for grp in groups:
        votes = run_batch(rb, w, cl, base, extras, hear, np.zeros((n, 1), bool), group=grp)
        assert len(votes.who) > 0 and len(votes.props) == 2
        ref = arms.tally(cl, votes)
        seen.append((ref.decided, ref.votes_received))
    assert seen[0][0] is False and seen[1][0] is True and seen[2] == seen[1]
    assert path != "in order" or ref.decided_at[0] == 1


@pytest.mark.gpu
def test_sharded_dissent_in_the_majoritys_bucket(rb, worlds, comm):
    """the dissenting cut falls into the same 12-bit bucket of the sum buffer as the winner's: the sum check cannot tell them
    apart and the refinement runs on its own"""
    n = 20_000
    w = worlds(n)
    base = W.pick_smallest(n, 5, W.SEED + 5)
    rng = np.random.default_rng(5)
    h_base = rb.proposal_fingerprint(np.sort(base))[0]
    extras = _pick_extras(rb, w, base, 1, rng, bucket_of=(lambda h: h >> 52, h_base))
    cl = rb.VirtualCluster(w.v, H, L)
    votes = run_batch(rb, w, cl, base, extras, _interleaved_hear(w, rng, 0.8), np.zeros((n, 1), bool))
    assert len(votes.props) == 2 and len({p[0] >> 52 for p in votes.props}) == 1
    ref = Arms(rb, w, "sharded", comm).tally(cl, votes)
    assert ref.decided
