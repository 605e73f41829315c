"""RAPID_DELIVERY_SHUFFLED_BATCHES on the CPU: the batch order P_g (include/rapid_b200.h) restated three times (NumPy, plain
Python, and the C++ next to the oracle's handlers) and checked to be a permutation with uniform small cases; the shuffled delivery over the oracle's handlers (tests/shuffled_ref.py) against
independent pyref.PyBatchHandlers fed batch by batch in each receiver's order."""
import itertools
import random

import numpy as np
import pytest

import pyref
import shuffled_ref as S
from helpers import OracleWorld
from test_oracle_vs_python_restatement import same_reports

K = 10
M64 = (1 << 64) - 1


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 15, 16, 17, 255, 256, 257, 4096, 10 ** 5])
def test_order_restatements_agree_and_permute(n):
    rng = random.Random(n)
    seeds = [0, 1, M64, rng.getrandbits(64)]
    gs = [0, 1, 7, 2 ** 40, rng.getrandbits(40)]
    for seed in seeds:
        many = S.batch_orders(seed, gs, n)
        for i, g in enumerate(gs):
            if n <= 4096 or (seed, g) == (seeds[-1], gs[-1]):      # the plain restatement is slow at 10^5
                assert many[i].tolist() == S.batch_order_plain(seed, g, n), (seed, g)
            assert many[i].tolist() == S.batch_order_oracle(seed, g, n), (seed, g)
            assert (np.sort(many[i]) == np.arange(n)).all(), (seed, g)


def test_order_of_five_is_uniform():
    from scipy.stats import chisquare
    rows = S.batch_orders(0x5EED, np.arange(10 ** 5), 5)
    index = {p: i for i, p in enumerate(itertools.permutations(range(5)))}
    counts = np.bincount([index[tuple(r)] for r in rows.tolist()], minlength=120)
    assert (counts > 0).all()
    assert chisquare(counts).pvalue > 1e-3


def test_order_depends_on_the_receiver_and_the_seed():
    a = S.batch_orders(3, np.arange(64), 40)
    assert len({tuple(r) for r in a.tolist()}) == 64
    assert (S.batch_orders(4, np.arange(64), 40) != a).any()


def _sequence(rng, w, n, n_batches):
    """random per-sender batches over a few crashed subjects and one joiner: duplicates, empty batches, UP and DOWN"""
    failed = rng.sample(range(n), rng.randint(1, 4))
    cells = [(w.view.getObserversOf(s)[k], s, k, pyref.DOWN) for s in failed for k in range(K)]
    cells = [c for c in cells if c[0] not in failed]
    cells += [(w.view.getExpectedObserversOf(n)[k], n, k, pyref.UP) for k in range(K)]
    cells += [rng.choice(cells) for _ in range(rng.randint(0, 8))]
    rng.shuffle(cells)
    cut = sorted(rng.sample(range(1, len(cells)), min(n_batches - 1, len(cells) - 1)))
    cut += [len(cells)] * (n_batches - 1 - len(cut))
    if n_batches > 2 and rng.random() < 0.5:
        cut[rng.randrange(len(cut))] = cut[0]                     # an empty batch
        cut.sort()
    off = np.array([0] + cut + [len(cells)], np.int64)
    src, dst, ring, st = (np.array(c, t) for c, t in zip(zip(*cells), (np.int32, np.int32, np.uint8, np.uint8)))
    return failed, src, dst, ring, st, off


@pytest.mark.parametrize("seed", range(25))
def test_shuffled_delivery_against_python_handlers(orc, seed):
    rng = random.Random(9100 + seed)
    n = rng.randint(12, 60)
    H, L = rng.choice([(9, 4), (8, 3), (8, 2)])
    w = OracleWorld(orc, n, K, n_joiners=1)
    cfg = w.view.getCurrentConfigurationId()
    R = rng.randint(1, n)
    base = rng.randint(0, n - R)
    sim = orc.ClusterSim(w.view, K, H, L, R, receiver_base=base)
    py = [pyref.PyBatchHandler(w.view, K, H, L) for _ in range(R)]
    for call in range(2):                                         # state carried over two calls
        failed, src, dst, ring, st, off = _sequence(rng, w, n, rng.randint(1, 12))
        cfgs = np.array([cfg if rng.random() < 0.95 else cfg ^ 1 for _ in src], np.int64)
        blocked = np.array([rng.random() < 0.2 for _ in range(R)], np.uint8) if seed % 2 else None
        oseed = rng.getrandbits(64)
        o_len, o_ann, o_props, o_in = S.apply_batches(sim, src, dst, ring, st, cfgs, off, blocked=blocked, order_seed=oseed,
                                                      receiver_base=base, threads=1)
        nb = len(off) - 1
        for r in range(R):
            got, ain = set(), -1
            if blocked is None or not blocked[r]:
                for b in S.batch_order_plain(oseed, base + r, nb):
                    if py[r].announcedProposal:
                        break
                    msgs = [(int(src[i]), int(dst[i]), int(st[i]), int(cfgs[i]), [int(ring[i])]) for i in range(off[b], off[b + 1])]
                    p = py[r].handleBatch(msgs)
                    if p:
                        got, ain = p, b
            assert (set(o_props[r]) if o_props[r] else set()) == got and o_len[r] == len(got), (seed, call, r)
            assert o_in[r] == ain and bool(o_ann[r]) == py[r].announcedProposal, (seed, call, r)
            assert sim.numProposals(r) == py[r].cd.getNumProposals()
            assert sim.updatesInProgress(r) == py[r].cd.updatesInProgress
            for t in failed + [n]:
                assert same_reports(sim.reportMask(r, t), py[r].cd.reportMask(t), H)

