"""The proposal census on the device (csrc/cd_census.cu, VirtualCluster.proposalCensus): every class's list, statuses, voters and
representative against the grouping of the oracle's per-receiver proposals; cls[r] against that grouping on every receiver;
every list against rapid_cd_get_proposal of its representative and its fingerprint against readOutputs(); distances from a cut
against set arithmetic; the refusals; the census at 10^5 and 10^6 receivers against the host grouping of readOutputs(); and
ClusterSimulation(proposal_census=True) against tests/censusref.py."""
import numpy as np
import pytest

import censusref
import shuffled_ref as S
from helpers import OracleWorld
from simref import CRASHED, flags, join, leave, random_hosts, run, same_run
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu
K, H, L = 10, 9, 4
N = 2000


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.fixture(scope="module", autouse=True)
def _free_worlds():
    """the views live as long as this module's tests"""
    yield
    _WORLD.clear()


@pytest.fixture(scope="module")
def world(orc, rb, _free_worlds):
    return _world(orc, rb, K, H, L)


# the census at other ring counts, each with H = K: the smallest K and the largest (a hi byte per receiver in the rows)
OTHER_KHL = [(3, 3, 1), (14, 14, 6)]
_WORLD = {}


def _world(orc, rb, Kx, Hx, Lx):
    if Kx not in _WORLD:
        w = OracleWorld(orc, N, Kx, n_joiners=8)
        v = rb.MembershipView.from_packed(Kx, *w.member_packed())
        v.registerJoiners(*w.joiner_endpoints())
        _WORLD[Kx] = dict(w=w, v=v, K=Kx, H=Hx, L=Lx, cfg=w.view.getCurrentConfigurationId(), obs=w.tables()[0], ring0=w.ring0(),
                          jobs=v.joinerTables())
    return _WORLD[Kx]


def per_sender(src, dst, ring, status):
    order = np.argsort(src, kind="stable")
    src, dst, ring, status = src[order], dst[order], ring[order], status[order]
    _, first = np.unique(src, return_index=True)
    return src, dst, ring, status, np.append(first, len(src)).astype(np.int64)


def groups(props):
    """per-receiver proposals (None: did not announce) -> [(frozenset, voters, lowest receiver)] in order of the lowest receiver,
    and the class of every receiver"""
    at, out, cls = {}, [], np.full(len(props), -1, np.int32)
    for r, p in enumerate(props):
        if p is None:
            continue
        k = frozenset(p)
        if k not in at:
            at[k] = len(out)
            out.append([k, 0, r])
        out[at[k]][1] += 1
        cls[r] = at[k]
    return out, cls


def check(rb, cl, props, cut=None, n_members=None):
    """the census of cl's last call against the per-receiver proposals props"""
    c = cl.proposalCensus(cut=cut)
    want, want_cls = groups(props)
    assert len(c) == len(want)
    out = cl.readOutputs()
    np.testing.assert_array_equal(c.classes(), want_cls)
    np.testing.assert_array_equal(c.classes() >= 0, out.proposal_len > 0)
    n_members = cl.view.n if n_members is None else n_members
    for i, (k, voters, rep) in enumerate(want):
        ids = c.entries(i)
        assert frozenset(ids.tolist()) == k and len(ids) == len(k) == c.length[i]
        assert (c.voters[i], c.representative[i]) == (voters, rep)
        assert ids.tolist() == cl.getProposal(rep)
        np.testing.assert_array_equal(c.statuses(i), np.where(ids < n_members, 1, 0))
        assert (int(c.hash[i]), int(c.hash2[i])) == (int(out.proposal_hash[rep]), int(out.proposal_hash2[rep]))
        assert (int(c.hash[i]), int(c.hash2[i])) == rb.proposal_fingerprint(ids)
        if cut is None:
            assert c.in_cut[i] == c.missing[i] == c.extra[i] == -1
        else:
            cs = frozenset(int(x) for x in cut)
            assert (c.missing[i], c.extra[i]) == (len(cs - k), len(k - cs))
    if len(want):
        assert c.classes_dev != 0
    return c


def oracle_sender(world, orc, seq, blocked, seed, R=N, base=0):
    """per-sender batches through the oracle's handlers, batch b with cell order seed + b -> per-receiver proposals of the call"""
    src, dst, ring, st, off = seq
    sim = orc.ClusterSim(world["w"].view, world["K"], world["H"], world["L"], R, receiver_base=base)
    props = [None] * R
    for b in range(len(off) - 1):
        sl = slice(off[b], off[b + 1])
        o_len, _, ids, o_off = sim.apply_batch(src[sl], dst[sl], ring[sl], st[sl], np.full(off[b + 1] - off[b], world["cfg"], np.int64),
                                               blocked=blocked, perm_seed=seed + b, threads=4)
        for r in np.nonzero(o_len)[0]:
            props[r] = ids[o_off[r]: o_off[r + 1]].tolist()
    return props


def c2(world, frac=0.01, seed=W.SEED):
    b = W.c2_simultaneous_crash(world["obs"], N, frac, seed)
    return per_sender(b.src, b.dst, b.ring, b.status), W.blocked_by_receiver(b.blocked, world["ring0"], 0, N)


# ---- against the oracle --------------------------------------------------------------------------------------------------------------
def test_bucketed_sender_batches_one_call(orc, rb, world):
    _sender_batches_one_call(orc, rb, world)


def _sender_batches_one_call(orc, rb, world):
    seq, blocked = c2(world)
    cl = rb.VirtualCluster(world["v"], world["H"], world["L"], kernel="bucketed")
    cl.handleBatches(world["cfg"], *seq, blocked=blocked, perm_seed=41, read_outputs=False)
    c = check(rb, cl, oracle_sender(world, orc, seq, blocked, 41))
    assert len(c) >= 1 and c.voters.sum() > N // 2


def test_bucketed_one_batch_per_call(orc, rb, world):
    """a batch per call: each census covers the receivers that announced in that call only"""
    (src, dst, ring, st, off), blocked = c2(world)
    cl = rb.VirtualCluster(world["v"], H, L, kernel="bucketed")
    sim = orc.ClusterSim(world["w"].view, K, H, L, N)
    seen = 0
    for b in range(len(off) - 1):
        sl = slice(off[b], off[b + 1])
        cl.handleBatch(world["cfg"], src[sl], dst[sl], ring[sl], st[sl], blocked=blocked, perm_seed=5 + b, read_outputs=False)
        o_len, _, ids, o_off = sim.apply_batch(src[sl], dst[sl], ring[sl], st[sl], np.full(off[b + 1] - off[b], world["cfg"], np.int64),
                                               blocked=blocked, perm_seed=5 + b, threads=4)
        props = [ids[o_off[r]: o_off[r + 1]].tolist() if o_len[r] else None for r in range(N)]
        if o_len.any() or b == len(off) - 2:
            check(rb, cl, props)
            seen += int((o_len > 0).sum())
    assert seen > N // 2


def test_joins_and_crashes_with_blocked_receivers(orc, rb, world):
    _joins_and_crashes(orc, rb, world)


def _joins_and_crashes(orc, rb, world):
    b = W.c5_churn(world["obs"], world["jobs"], N, 6, 8, seed=11)
    blocked = W.blocked_by_receiver(b.blocked, world["ring0"], 0, N)
    assert blocked.any()
    seq = per_sender(b.src, b.dst, b.ring, b.status)
    cl = rb.VirtualCluster(world["v"], world["H"], world["L"], kernel="bucketed")
    cl.handleBatches(world["cfg"], *seq, blocked=blocked, perm_seed=3, read_outputs=False)
    c = check(rb, cl, oracle_sender(world, orc, seq, blocked, 3))
    assert (c.status == 0).any() and (c.status == 1).any()                      # UP (joiners) and DOWN entries
    assert (c.classes()[blocked.astype(bool)] == -1).all()


def test_shuffled_c2_many_proposals(orc, rb, world):
    seq, blocked = c2(world, 0.002)                               # 4 crashed: receivers announce 9 different subsets
    cl = rb.VirtualCluster(world["v"], H, L, kernel="sweep")
    cl.handleBatches(world["cfg"], *seq, blocked=blocked, batch_order_seed=77, read_outputs=False)
    sim = orc.ClusterSim(world["w"].view, K, H, L, N)
    _, _, props, _ = S.apply_batches(sim, *seq[:4], world["cfg"], seq[4], blocked=blocked, order_seed=77)
    c = check(rb, cl, props)
    assert len(c) >= 3
    # the decided-cut, disjoint and empty cuts on the same call
    m = int(np.argmax(c.voters))
    check(rb, cl, props, cut=c.entries(m))
    universe = set(range(N + 8))
    disjoint = sorted(universe - set(c.ids.tolist()))[:50]
    check(rb, cl, props, cut=disjoint)
    e = check(rb, cl, props, cut=[])
    np.testing.assert_array_equal(e.in_cut, 0)


def test_shard_second_call_and_clear(orc, rb, world):
    _shard_second_call_and_clear(orc, rb, world)


@pytest.mark.parametrize("case", ["sender-batches", "joins-and-crashes", "shard"])
@pytest.mark.parametrize("Kx,Hx,Lx", OTHER_KHL, ids=["K%d" % k for k, _, _ in OTHER_KHL])
def test_census_at_other_ring_counts(orc, rb, Kx, Hx, Lx, case):
    """the sender-batches call, joins and crashes with blocked receivers, and the shard's two calls at K = 3 and K = 14"""
    world = _world(orc, rb, Kx, Hx, Lx)
    {"sender-batches": _sender_batches_one_call, "joins-and-crashes": _joins_and_crashes,
     "shard": _shard_second_call_and_clear}[case](orc, rb, world)


def _shard_second_call_and_clear(orc, rb, world):
    (src, dst, ring, st, off), blocked = c2(world, 0.005, seed=5)
    half = len(off) // 2
    first = (src[: off[half]], dst[: off[half]], ring[: off[half]], st[: off[half]], off[: half + 1])
    second = (src[off[half]:], dst[off[half]:], ring[off[half]:], st[off[half]:], off[half:] - off[half])
    base, R = 700, 500
    cl = rb.VirtualCluster(world["v"], world["H"], world["L"], n_receivers=R, receiver_begin=base, kernel="sweep")
    sim = orc.ClusterSim(world["w"].view, world["K"], world["H"], world["L"], R, receiver_base=base)
    bl = blocked[base: base + R]
    announced = 0
    for i, part in enumerate((first, second)):
        cl.handleBatches(world["cfg"], *part, blocked=bl, batch_order_seed=1 + i, read_outputs=False)
        _, _, props, _ = S.apply_batches(sim, *part[:4], world["cfg"], part[4], blocked=bl, order_seed=1 + i, receiver_base=base)
        c = check(rb, cl, props)
        assert (c.representative < R).all()
        announced += int(c.voters.sum())
    assert announced > 0
    cl.clear()
    c = cl.proposalCensus()
    assert len(c) == 0 and len(c.ids) == 0 and c.list_off.tolist() == [0]
    assert (c.classes() == -1).all()


# ---- refusals ------------------------------------------------------------------------------------------------------------------
def _snapshot(c):
    return [a.copy() for a in (c.hash, c.hash2, c.length, c.voters, c.representative, c.in_cut, c.list_off, c.ids, c.status)]


def _reread(rb, cl, nc, ne, cut_len):
    """the handle's current census, read again"""
    c = rb.cut_detector.ProposalCensus(cl, nc, ne, cut_len)
    return _snapshot(c), c.classes()


def test_refusals_leave_the_previous_census(rb):
    N_ = rb._native
    n = 60
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    obs, _ = v.tables()
    b = W.c2_simultaneous_crash(obs, n, 0.1, 3)
    blocked = W.blocked_by_receiver(b.blocked, np.asarray(v.getRing(0)), 0, n)
    fresh = rb.VirtualCluster(v, H, L)
    with pytest.raises(N_.RapidError) as e:
        fresh.proposalCensus()
    assert e.value.code == N_.EINVAL and "no batch" in str(e.value)
    cl = rb.VirtualCluster(v, H, L)
    cl.handleBatch(0, b.src, b.dst, b.ring, b.status, blocked=blocked, read_outputs=False)
    cut = sorted(int(x) for x in b.expected_cut)
    c = cl.proposalCensus(cut=cut)
    assert len(c) >= 1
    before, before_cls = _snapshot(c), c.classes()
    outs = cl.readOutputs()
    for bad in ([n + 5], [-1], [cut[0], cut[0]]):
        with pytest.raises(N_.RapidError) as e:
            cl.proposalCensus(cut=bad)
        assert e.value.code == N_.EINVAL
    rc = N_.lib().rapid_cd_proposal_census(cl._h, None, 3, None, None)               # a length without ids
    assert rc == N_.EINVAL
    raw = rb.MultiNodeCutDetector(v, H, L, n_detectors=4)
    rc = N_.lib().rapid_cd_proposal_census(raw._h, None, 0, None, None)
    assert rc == N_.EINVAL and "RAW" in N_.last_error()
    after, after_cls = _reread(rb, cl, len(c), len(c.ids), len(cut))
    for x, y in zip(before, after):
        np.testing.assert_array_equal(x, y)
    np.testing.assert_array_equal(before_cls, after_cls)
    now = cl.readOutputs()
    for f in ("proposal_hash", "proposal_hash2", "proposal_len", "announced"):
        np.testing.assert_array_equal(getattr(outs, f), getattr(now, f))
    v.applyCut(cut)                                                              # the members change: the handle predates them
    with pytest.raises(N_.RapidError) as e:
        cl.proposalCensus()
    assert e.value.code == N_.EINVAL and "members changed" in str(e.value)
    after, _ = _reread(rb, cl, len(c), len(c.ids), len(cut))
    for x, y in zip(before, after):
        np.testing.assert_array_equal(x, y)


# ---- scale ---------------------------------------------------------------------------------------------------------------------
def host_check(rb, cl, c, sample=40):
    """the census against the host grouping of readOutputs(), and sampled lists against getProposal of their representative"""
    out = cl.readOutputs()
    now = np.nonzero(out.proposal_len > 0)[0]
    fps = {}
    for r in now.tolist():
        fps.setdefault((int(out.proposal_hash[r]), int(out.proposal_hash2[r]), int(out.proposal_len[r])), []).append(r)
    assert len(c) == len(fps)
    got = {(int(c.hash[i]), int(c.hash2[i]), int(c.length[i])): i for i in range(len(c))}
    assert set(got) == set(fps)
    cls = c.classes()
    for fp, rs in fps.items():
        i = got[fp]
        assert c.voters[i] == len(rs) and c.representative[i] == rs[0]
        assert (cls[rs] == i).all()
    assert (cls >= 0).sum() == len(now)
    assert (np.diff(c.representative) > 0).all()
    for i in list(range(len(c)))[:: max(1, len(c) // sample)]:
        assert c.entries(i).tolist() == cl.getProposal(int(c.representative[i]))


def test_hundred_thousand_receivers_shuffled(rb):
    n = 100_000
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    obs, _ = v.tables()
    b = W.c2_simultaneous_crash(obs, n, 1e-4, 17)                # 10 crashed: a dozen different proposals
    blocked = W.blocked_by_receiver(b.blocked, np.asarray(v.getRing(0)), 0, n)
    cl = rb.VirtualCluster(v, H, L, kernel="sweep")
    cl.handleBatches(0, *per_sender(b.src, b.dst, b.ring, b.status), blocked=blocked, batch_order_seed=5, read_outputs=False)
    c = cl.proposalCensus()
    host_check(rb, cl, c)
    assert len(c) >= 2


def test_million_receivers_sender_mode(rb):
    n, nj = 1_000_000, 5_000
    v = rb.MembershipView.from_packed(K, *W.packed_endpoints(0, n))
    v.registerJoiners(*W.endpoints(n, nj))
    obs, _ = v.tables()
    b = W.c5_churn(obs, v.joinerTables(), n, n // 200, nj)
    blocked = W.blocked_by_receiver(b.blocked, np.asarray(v.getRing(0)), 0, n)
    cl = rb.VirtualCluster(v, H, L, max_subjects=len(b.expected_cut) + 64)
    cl.handleBatch(0, None, b.dst, b.ring, b.status, blocked=blocked, read_outputs=False)
    c = cl.proposalCensus(cut=np.asarray(b.expected_cut, np.int32))
    host_check(rb, cl, c, sample=4)
    m = int(np.argmax(c.voters))
    assert c.missing[m] == c.extra[m] == 0 and c.length[m] == len(b.expected_cut)
    assert (c.statuses(m) == 0).sum() == nj


# ---- through the cluster simulation ------------------------------------------------------------------------------------------------
TIMES = ("detect_ms", "classic_ms", "view_change_ms", "handles_ms", "device_ms", "host_ms")


def make(orc, rb, n, seed, nj=0, **kw):
    ref = censusref.CensusOracleSimulation(orc, n, seed=seed, n_joiners=nj, **kw)
    on = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed, proposal_census=True, **kw)
    off = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed, **kw)
    return ref, on, off


def same_without_census(on, off):
    """every record of the run with the census equals the run without it, but for census, agreement and the timings"""
    for a, b in ((on.intervals, off.intervals), (on.history, off.history)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            assert {k: v for k, v in x.items() if k not in TIMES + ("census", "agreement")} == \
                   {k: v for k, v in y.items() if k not in TIMES}


def census_consistent(s):
    for r in s.intervals:
        assert ("census" in r) == (r["announced"] > 0)
        if "census" in r:
            assert sum(c["voters"] for c in r["census"]) == r["announced"] and len(r["census"]) == r["proposals"]
    for h in s.history:
        assert sum(c["decided"] for c in h["census"]) == 1 and len(h["census"]) == h["distinct_proposals"]
        d = [c for c in h["census"] if c["decided"]][0]
        assert d["missing"] == d["extra"] == 0 and d["size"] == len(h["cut"])
        assert 0 < h["agreement"] <= 1


@pytest.mark.parametrize("batch_order", ["sender", "shuffled"])
@pytest.mark.parametrize("n,f,seed,nj", [(5, 1, 1, 0), (50, 12, 3, 0), (50, 16, 6, 0), (30, 5, 13, 10), (50, 12, 12, 0)])
def test_cluster_scenarios(orc, rb, batch_order, n, f, seed, nj):
    failing = [2] if n == 5 else random_hosts(n, f, seed)
    sims = make(orc, rb, n, seed, nj, batch_order=batch_order)
    join(sims, range(n, n + nj))
    flags(sims, failing, CRASHED)
    run(sims, 30)
    same_run(sims[0], sims[1])
    same_without_census(sims[1], sims[2])
    census_consistent(sims[1])
    if (batch_order, n, seed) == ("shuffled", 50, 12):                          # three cuts announced, the classic round decides
        h = sims[1].history[0]
        assert len(h["census"]) == 3 and h["path"] == "classic" and h["agreement"] < 1


@pytest.mark.parametrize("batch_order", ["sender", "shuffled"])
def test_graceful_leave(orc, rb, batch_order):
    sims = make(orc, rb, 50, 31, batch_order=batch_order)
    leave(sims, [4, 17])
    run(sims)
    same_run(sims[0], sims[1])
    same_without_census(sims[1], sims[2])
    census_consistent(sims[1])


@pytest.mark.parametrize("n,batch_order", [(1_000, "sender"), (1_000, "shuffled"), (10_000, "sender"), (10_000, "shuffled")])
def test_one_percent_crashed(orc, rb, n, batch_order):
    seed = 21
    sims = make(orc, rb, n, seed, batch_order=batch_order)
    flags(sims, W.pick_smallest(n, n // 100, seed).tolist(), CRASHED)
    run(sims, 15)
    same_run(sims[0], sims[1])
    same_without_census(sims[1], sims[2])
    census_consistent(sims[1])


def test_conflict_census_device_and_oracle_agree(orc, rb):
    """profiles/conflict_census.py --reps 2: the device and the oracle print the same table"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = os.path.join(root, "profiles", "conflict_census.py")
    outs = []
    for extra in ([], ["--oracle"]):
        r = subprocess.run([sys.executable, script, "--reps", "2"] + extra, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(json.loads(r.stdout.strip().splitlines()[-1])["table"])
    assert outs[0] == outs[1]
    assert any(row["disagree"] > 0 for row in outs[0])

