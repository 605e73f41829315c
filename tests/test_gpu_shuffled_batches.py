"""RAPID_DELIVERY_SHUFFLED_BATCHES on the device: the sweep kernel's per-receiver batch order (k_sweep<true>) against the oracle's
literal handlers walked in the same order (tests/shuffled_ref.py) receiver by receiver; the flag's refusals; and
ClusterSimulation(batch_order="shuffled") against tests/simref.py, record by record."""
import numpy as np
import pytest

import shuffled_ref as S
from helpers import OracleWorld
from simref import CRASHED, flags, join, leave, make, random_hosts, run, same_run
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu
K, H, L = 10, 9, 4
N = 2000


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


@pytest.fixture(scope="module")
def world(orc, rb):
    w = OracleWorld(orc, N, K, n_joiners=8)
    v = rb.MembershipView.from_packed(K, *w.member_packed())
    v.registerJoiners(*w.joiner_endpoints())
    return dict(w=w, v=v, cfg=w.view.getCurrentConfigurationId(), obs=w.tables()[0], ring0=w.ring0(), jobs=v.joinerTables())


def per_sender(src, dst, ring, status):
    """one batch per sender, senders ascending, cells of a sender in their given order"""
    order = np.argsort(src, kind="stable")
    src, dst, ring, status = src[order], dst[order], ring[order], status[order]
    _, first = np.unique(src, return_index=True)
    return src, dst, ring, status, np.append(first, len(src)).astype(np.int64)


def compare(rb, world, cl, sim, seq, blocked, seed, base=0):
    src, dst, ring, st, off = seq
    o_len, o_ann, o_props, o_in = S.apply_batches(sim, src, dst, ring, st, world["cfg"], off, blocked=blocked, order_seed=seed,
                                                  receiver_base=base)
    res, ain = cl.handleBatches(world["cfg"], src, dst, ring, st, off, blocked=blocked, batch_order_seed=seed)
    np.testing.assert_array_equal(res.proposal_len, o_len)
    np.testing.assert_array_equal(res.announced, o_ann)
    np.testing.assert_array_equal(ain, o_in)
    for r in np.nonzero(o_len)[0]:
        assert (res.proposal_hash[r], res.proposal_hash2[r]) == rb.proposal_fingerprint(o_props[r]), r
    who = np.nonzero(o_len)[0]
    for r in who[:: max(1, len(who) // 8)][:8]:
        assert cl.getProposal(int(r)) == o_props[r], r
    live = np.nonzero(o_ann == 0)[0]
    for r in live[:: max(1, len(live) // 8)][:8]:
        for subj, m in cl.debugMasks(int(r)).items():
            assert sim.reportMask(int(r), int(subj)) == m, (subj, r)
        assert cl.debugCounters(int(r))[0] == sim.updatesInProgress(int(r))
    return o_len, o_in


def c2(world, frac=0.01, seed=W.SEED):
    b = W.c2_simultaneous_crash(world["obs"], N, frac, seed)
    blocked = W.blocked_by_receiver(b.blocked, world["ring0"], 0, N)
    return per_sender(b.src, b.dst, b.ring, b.status), blocked


def test_c2_crashes_as_sender_batches(orc, rb, world):
    seq, blocked = c2(world)
    assert len(seq[4]) > 150                                      # ~200 sender batches
    cl = rb.VirtualCluster(world["v"], H, L, kernel="sweep")
    sim = orc.ClusterSim(world["w"].view, K, H, L, N)
    o_len, o_in = compare(rb, world, cl, sim, seq, blocked, seed=77)
    assert (o_len > 0).sum() > N // 2 and len(set(o_in[o_in >= 0].tolist())) > 1   # receivers announce at different batches


def test_two_calls_carry_state_and_a_shard(orc, rb, world):
    (src, dst, ring, st, off), blocked = c2(world, 0.005, seed=5)
    half = len(off) // 2
    first = (src[: off[half]], dst[: off[half]], ring[: off[half]], st[: off[half]], off[: half + 1])
    second = (src[off[half]:], dst[off[half]:], ring[off[half]:], st[off[half]:], off[half:] - off[half])
    base, R = 700, 500                                            # receiver_begin != 0
    cl = rb.VirtualCluster(world["v"], H, L, n_receivers=R, receiver_begin=base, kernel="sweep")
    sim = orc.ClusterSim(world["w"].view, K, H, L, R, receiver_base=base)
    bl = blocked[base: base + R]
    compare(rb, world, cl, sim, first, bl, seed=1, base=base)
    compare(rb, world, cl, sim, second, bl, seed=2, base=base)


def test_joins_and_crashes(orc, rb, world):
    nj = 8
    b = W.c5_churn(world["obs"], world["jobs"], N, 6, nj, seed=11)
    blocked = W.blocked_by_receiver(b.blocked, world["ring0"], 0, N)
    cl = rb.VirtualCluster(world["v"], H, L, kernel="sweep")
    sim = orc.ClusterSim(world["w"].view, K, H, L, N)
    o_len, _ = compare(rb, world, cl, sim, per_sender(b.src, b.dst, b.ring, b.status), blocked, seed=3)
    assert o_len.max() > nj


def test_one_batch_equals_the_unflagged_call(rb, world):
    (src, dst, ring, st, _), blocked = c2(world)
    off = np.array([0, len(dst)], np.int64)
    a = rb.VirtualCluster(world["v"], H, L, kernel="sweep")
    b = rb.VirtualCluster(world["v"], H, L, kernel="sweep")
    ra, ia = a.handleBatches(world["cfg"], src, dst, ring, st, off, blocked=blocked, batch_order_seed=9)
    rb_, ib = b.handleBatches(world["cfg"], src, dst, ring, st, off, blocked=blocked)
    for f in ("proposal_hash", "proposal_hash2", "proposal_len", "announced"):
        np.testing.assert_array_equal(getattr(ra, f), getattr(rb_, f))
    np.testing.assert_array_equal(ia, ib)


def _state(cl, rs):
    return [(cl.debugMasks(r), cl.debugCounters(r)) for r in rs]


def test_refusals_change_nothing(rb, world):
    N_ = rb._native
    (src, dst, ring, st, off), blocked = c2(world)
    cfg = world["cfg"]
    rs = [0, 5, 999]
    for kernel in ("sweep", "bucketed"):
        cl = rb.VirtualCluster(world["v"], H, L, kernel=kernel)
        cl.handleBatch(cfg, src[: off[3]], dst[: off[3]], ring[: off[3]], st[: off[3]])   # some state to keep
        before = (_state(cl, rs), cl.readOutputs().proposal_len.copy(), cl.lastPath())
        calls = [lambda: cl.handleBatches(cfg, src, dst, ring, st, off, batch_order_seed=1, perm_seed=2),
                 lambda: cl.handleBatches(cfg, src, dst, ring, st, off, batch_order_seed=1,
                                          bitmap=np.full((len(dst), (N + 31) // 32), 0xFFFFFFFF, np.uint32))]
        if kernel == "bucketed":
            calls.append(lambda: cl.handleBatches(cfg, src, dst, ring, st, off, batch_order_seed=1))
        else:                                                     # PERMUTED needs a bucketed handle: refused before k_prepare runs
            calls.append(lambda: cl.handleBatch(cfg, src, dst, ring, st, perm_seed=3))
        for i, call in enumerate(calls):
            with pytest.raises(N_.RapidError) as e:
                call()
            want = N_.EUNSUPPORTED if i == 2 else N_.EINVAL
            assert e.value.code == want, (kernel, i, str(e.value))
            if i == 2:
                assert ("RAPID_CD_SWEEP" if kernel == "bucketed" else "needs a bucketed handle") in str(e.value)
        d = N_.Delivery()
        d.flags, d.perm_seed = N_.DELIVERY_SHUFFLED_BATCHES, 1
        rc = N_.lib().rapid_cd_apply_batch(cl._h, int(cfg), len(dst), N_.ptr(src), N_.ptr(dst), N_.ptr(ring), N_.ptr(st), None,
                                           __import__("ctypes").byref(d), None, None, None, None)
        assert rc == N_.EINVAL
        assert _state(cl, rs) == before[0]
        np.testing.assert_array_equal(cl.readOutputs().proposal_len, before[1])
        assert cl.lastPath() == before[2], kernel
    raw = rb.MultiNodeCutDetector(world["v"], H, L, n_detectors=4)
    for i in range(0, 40, 7):
        raw.aggregateForProposal(int(src[i]), int(dst[i]), int(st[i]), [int(ring[i])], detector=i % 4)
    raw_state = [(rb.VirtualCluster.debugMasks(raw, r), rb.VirtualCluster.debugCounters(raw, r), raw.getNumProposals(r))
                 for r in range(4)]
    d = N_.Delivery()
    d.flags, d.perm_seed = N_.DELIVERY_SHUFFLED_BATCHES, 1
    rc = N_.lib().rapid_cd_apply_batches(raw._h, int(cfg), len(dst), N_.ptr(src), N_.ptr(dst), N_.ptr(ring), N_.ptr(st), None,
                                         len(off) - 1, N_.ptr(off), __import__("ctypes").byref(d), None, None, None, None, None)
    assert rc == N_.EUNSUPPORTED and "RAPID_CD_SWEEP" in N_.last_error()
    assert raw_state == [(rb.VirtualCluster.debugMasks(raw, r), rb.VirtualCluster.debugCounters(raw, r), raw.getNumProposals(r))
                         for r in range(4)]
    assert any(m for m, _, _ in raw_state)


# ---- ClusterSimulation(batch_order="shuffled") against simref ---------------------------------------------------------------------
@pytest.mark.parametrize("n,f,seed,flag,nj", [(5, 1, 1, 1, 0), (50, 12, 3, 1, 0), (50, 16, 6, 1, 0), (50, 10, 9, 2, 0),
                                               (30, 5, 13, 1, 10), (1000, 10, 21, 1, 0)])
def test_cluster_scenarios_shuffled(orc, rb, n, f, seed, flag, nj):
    failing = [2] if n == 5 else random_hosts(n, f, seed)
    ref, dev = sims = make(orc, rb, n, seed, nj, batch_order="shuffled")
    join(sims, range(n, n + nj))
    flags(sims, failing, flag)
    a, b = ref.run(30), dev.run(30)
    assert a["converged"] == b["converged"]
    same_run(ref, dev)


@pytest.mark.parametrize("n,f,seed,nj", [(50, 16, 6, 0), (30, 5, 13, 10)])
def test_cluster_scenarios_sender_mode_records(orc, rb, n, f, seed, nj):
    """the new record keys in the default mode, against simref(batch_order="sender")"""
    failing = random_hosts(n, f, seed)
    ref, dev = sims = make(orc, rb, n, seed, nj, batch_order="sender")
    join(sims, range(n, n + nj))
    flags(sims, failing, CRASHED)
    run(sims)
    same_run(ref, dev)


def test_ten_thousand_nodes_shuffled(orc, rb):
    n, seed = 10_000, 21
    failing = W.pick_smallest(n, n // 100, seed).tolist()
    ref, dev = sims = make(orc, rb, n, seed, batch_order="shuffled")
    flags(sims, failing, CRASHED)
    run(sims, 15)
    same_run(ref, dev)


def test_leave_shuffled(orc, rb):
    ref, dev = sims = make(orc, rb, 50, 31, batch_order="shuffled")
    leave(sims, [4, 17])
    run(sims)
    same_run(ref, dev)
    assert 4 not in dev.members() and 17 not in dev.members()


def test_conflicting_proposals_go_to_the_classic_round(orc, rb):
    """the behaviour the mode exists for: receivers that meet the batches in different orders announce three different cuts, no
    fast quorum forms, and the classic round decides"""
    n, seed = 50, 12
    failing = random_hosts(n, 12, seed)
    ref, dev = sims = make(orc, rb, n, seed, batch_order="shuffled")
    flags(sims, failing, CRASHED)
    run(sims)
    same_run(ref, dev)
    assert dev.history[0]["distinct_proposals"] == 3 and dev.history[0]["path"] == "classic"
    assert max(r["proposals"] for r in dev.intervals) >= 2


def test_conflict_study_device_and_oracle_agree(orc, rb):
    """profiles/conflict_study.py on a reduced grid of 2 repetitions: the device and the oracle print the same table"""
    import os
    import subprocess
    import sys
    import json
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    tables = []
    with tempfile.TemporaryDirectory() as d:
        for extra in ([], ["--oracle"]):
            out = os.path.join(d, "t%d.json" % len(tables))
            subprocess.check_call([sys.executable, os.path.join(root, "profiles", "conflict_study.py"), "--reps", "2", "--out", out]
                                  + extra)
            tables.append(json.load(open(out))["table"])
    assert tables[0] == tables[1]
    assert len(tables[0]) == 20 and any(r["conflict"] > 0 for r in tables[0])
