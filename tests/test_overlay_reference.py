"""tests/overlayref.py — the plain reference the device's overlay spectrum is compared with — pinned before anything leans on
it: its dense and sparse solvers agree, the matrix has the rows the definition gives it, a case with a closed form comes out
exactly, and the graph built from the oracle view's getObserversOf / getSubjectsOf is the one built from its rings."""
import numpy as np
import pytest

import overlayref as R
from helpers import OracleWorld
from rapid_b200 import workloads as W


def random_rings(n, K, seed):
    rng = np.random.default_rng(seed)
    return [rng.permutation(n) for _ in range(K)]


def test_dense_and_sparse_solvers_agree():
    rings = random_rings(500, 10, 1)
    d, s = R.overlay_lambdas(rings, dense=True), R.overlay_lambdas(rings, dense=False)
    assert d == pytest.approx(s, abs=1e-6)
    assert 2 * 10 * 0.3 < d[0] < 2 * 10 * 0.6 and -2 * 10 * 0.6 < d[1] < -2 * 10 * 0.3


@pytest.mark.parametrize("n,K", [(3, 3), (50, 10), (500, 14)])
def test_rows_sum_to_2K_and_the_matrix_is_symmetric(n, K):
    A = R.overlay_matrix(random_rings(n, K, n + K))
    assert (np.asarray(A.sum(axis=1)).ravel() == 2 * K).all()
    assert abs(A - A.T).max() == 0
    w = np.linalg.eigvalsh(A.toarray())
    assert w[-1] == pytest.approx(2 * K, abs=1e-9)


@pytest.mark.parametrize("n,K", [(7, 3), (50, 10), (501, 4)])
def test_K_copies_of_one_ring_give_the_cycle_graph(n, K):
    ring = random_rings(n, 1, n)[0]
    lam2, lmin = R.overlay_lambdas([ring] * K)
    assert lam2 == pytest.approx(2 * K * np.cos(2 * np.pi / n), abs=1e-9)
    assert lmin == pytest.approx(2 * K * np.cos(2 * np.pi * (n // 2) / n), abs=1e-9)
    A = R.overlay_matrix([ring] * K)
    assert set(A.data.tolist()) == {float(K)}                   # multiplicities are kept, not collapsed


def test_the_start_vector_is_what_the_header_says():
    x = R.start_vector(1000, 5)
    assert abs(x.sum()) < 1e-12 and np.linalg.norm(x) == pytest.approx(1.0, abs=1e-14)
    assert (R.splitmix64(np.uint64(5) + np.arange(3, dtype=np.uint64)) == W.splitmix64(np.arange(5, 8, dtype=np.uint64))).all()
    a, b = R.lanczos(R.overlay_matrix(random_rings(300, 10, 2)), 0, 60)
    hi, lo, res = R.ritz_ends(a, b)
    want = R.overlay_lambdas(random_rings(300, 10, 2))
    assert abs(hi - want[0]) <= res + 1e-9 and abs(lo - want[1]) <= res + 1e-9 and res < 0.05


def _relabelled(view, K):
    """(rings, obs, subj) of an oracle view with its members renumbered 0..n-1 in tag order"""
    tags = sorted(view.getRing(0))
    idx = {t: i for i, t in enumerate(tags)}
    rings = [[idx[t] for t in view.getRing(k)] for k in range(K)]
    obs = [[idx[t] for t in view.getObserversOf(m)] for m in tags]
    subj = [[idx[t] for t in view.getSubjectsOf(m)] for m in tags]
    return rings, obs, subj


def test_graph_from_observer_lists_equals_graph_from_rings(orc):
    n, K, nj = 200, 10, 20
    w = OracleWorld(orc, n, K, n_joiners=nj)
    for round_ in range(2):
        rings, obs, subj = _relabelled(w.view, K)
        A, B = R.overlay_matrix(rings), R.matrix_from_tables(obs, subj)
        assert A.shape == B.shape and abs(A - B).max() == 0
        assert (np.asarray(A.sum(axis=1)).ravel() == 2 * K).all()
        if round_ == 0:                                             # a ringDelete / ringAdd round, then once more
            for t in range(0, n, 3):
                w.view.ringDelete(t)
            hi, lo = W.node_ids(n, nj)
            for j in range(nj):
                w.view.ringAdd(n + j, (int(hi[j]), int(lo[j])))
            assert w.view.getMembershipSize() == n - len(range(0, n, 3)) + nj


def test_a_small_view_keeps_multiplicities(orc):
    """with 4 members and 10 rings every node observes some node on several rings: the entries of A count them"""
    K = 10
    w = OracleWorld(orc, 4, K)
    rings, obs, subj = _relabelled(w.view, K)
    A = R.overlay_matrix(rings)
    assert A.max() > 1 and abs(A - R.matrix_from_tables(obs, subj)).max() == 0
