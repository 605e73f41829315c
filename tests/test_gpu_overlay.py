"""rapid_view_overlay_spectrum (rapid_b200/csrc/overlay.cu) through the C ABI against tests/overlayref.py on the rings read back from
the device view: the two reported eigenvalues within the reported residual, exhausted Krylov spaces, multiplicities, the trivial
eigenvalue never reported, reproducibility, the view after applyCut, 10^6 nodes, refusals, and ClusterSimulation's option."""
import numpy as np
import pytest

import overlayref as R
from simref import CRASHED
from rapid_b200 import workloads as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rb():
    import rapid_b200
    return rapid_b200


def make_view(rb, n, K, first=0):
    return rb.MembershipView.from_packed(K, *W.packed_endpoints(first, n))


def rings_of(view):
    return [view.getRing(k) for k in range(view.K)]


def within(sp, want, K, A=None):
    """The residual bounds the distance from each reported value to SOME eigenvalue of A (checked against the whole spectrum where A
    is given); Ritz values lie inside the spectrum, so lambda2 approaches the true one from below and lambda_min from above.  At the
    edge of a dense bulk the nearest eigenvalue need not be the extreme one: the extreme one is allowed twice the residual."""
    eps = 1e-9 * 2 * K
    assert -eps <= want[0] - sp.lambda2 <= max(2 * sp.residual, eps), (sp, want)
    assert -eps <= sp.lambda_min - want[1] <= max(2 * sp.residual, eps), (sp, want)
    if A is not None:
        w = np.linalg.eigvalsh(A.toarray())[:-1]
        assert abs(w - sp.lambda2).min() <= sp.residual + eps and abs(w - sp.lambda_min).min() <= sp.residual + eps, sp
    if want[0] < 2 * K * (1 - 1e-6):
        assert sp.lambda2 < 2 * K * (1 - 1e-6)                          # 2K never comes back
    assert sp.lambda_ == max(abs(sp.lambda2), abs(sp.lambda_min)) and sp.ratio == sp.lambda_ / (2 * K)


@pytest.mark.parametrize("K", [3, 10, 14])
@pytest.mark.parametrize("n", [3, 4, 50, 1000, 20000])
def test_against_the_reference(rb, n, K):
    view = make_view(rb, n, K)
    sp = view.overlaySpectrum()
    assert np.isfinite([sp.lambda2, sp.lambda_min, sp.residual]).all() and 1 <= sp.steps <= min(256, n - 1)
    within(sp, R.overlay_lambdas(rings_of(view)), K, R.overlay_matrix(rings_of(view)) if n <= R.DENSE_LIMIT else None)
    if n >= 50:
        assert sp.residual <= 1e-3 * 2 * K, sp                          # converged at the default tolerance
    assert sp.device_ms > 0


@pytest.mark.parametrize("K", [3, 10, 14])
@pytest.mark.parametrize("n", [3, 4, 5])
def test_small_views_exhaust_the_krylov_space(rb, n, K):
    view = make_view(rb, n, K)
    sp = view.overlaySpectrum(seed=n, tol=1e-12, max_steps=512)
    want = R.overlay_lambdas(rings_of(view))
    assert np.isfinite([sp.lambda2, sp.lambda_min, sp.residual]).all()
    assert sp.lambda2 == pytest.approx(want[0], abs=1e-9) and sp.lambda_min == pytest.approx(want[1], abs=1e-9)
    assert sp.steps <= n - 1 and sp.residual <= 1e-9


@pytest.mark.parametrize("K", [10, 14])
def test_two_steps_follow_the_documented_start_vector_and_count_multiplicities(rb, K):
    """with max_steps = 2 the Ritz values are a function of alpha_1, beta_1, alpha_2 only (and the residual of beta_2): the reference
    restates the start vector and two steps with its own matrix.  On 50 nodes some node observes another on several rings; a kernel
    that counted it once would differ in alpha_1 already."""
    view = make_view(rb, 50, K)
    A = R.overlay_matrix(rings_of(view))
    assert A.max() > 1, "no repeated observer in this view: the case would not tell"
    for seed in (0, 7, 2 ** 63 + 11):
        sp = view.overlaySpectrum(seed=seed, tol=1e-12, max_steps=2)
        hi, lo, res = R.ritz_ends(*R.lanczos(A, seed, 2))
        assert sp.steps == 2
        assert sp.lambda2 == pytest.approx(hi, abs=1e-12 * 2 * K) and sp.lambda_min == pytest.approx(lo, abs=1e-12 * 2 * K)
        assert sp.residual == pytest.approx(res, abs=1e-10 * 2 * K)
        collapsed = A.copy()
        collapsed.data[:] = 1.0
        chi, clo, _ = R.ritz_ends(*R.lanczos(collapsed, seed, 2))
        assert abs(chi - hi) > 1e-6 or abs(clo - lo) > 1e-6


@pytest.mark.parametrize("n,K", [(1000, 10), (30000, 7)])
def test_same_seed_same_bits_other_seed_within_the_residuals(rb, n, K):
    view = make_view(rb, n, K)
    a, b, c = view.overlaySpectrum(seed=3), view.overlaySpectrum(seed=3), view.overlaySpectrum(seed=4)
    assert a[:4] == b[:4] and a.lambda_ == b.lambda_                     # everything but the timing, bit for bit
    assert abs(a.lambda2 - c.lambda2) <= a.residual + c.residual and abs(a.lambda_min - c.lambda_min) <= a.residual + c.residual
    assert (a.lambda2, a.lambda_min) != (c.lambda2, c.lambda_min)


def test_after_apply_cut(rb):
    """10,000 nodes, 30 % removed and 500 joiners admitted: the spectrum of the view updated in place equals that of a view built
    afresh from the surviving endpoints (ids equal, so bit for bit), and the reference's on the rings read back"""
    n, K, nj = 10000, 10, 500
    view = make_view(rb, n, K)
    hosts, ports = W.endpoints(n, nj)
    joiners = view.registerJoiners(hosts, ports)
    gone = W.pick_smallest(n, 3000, 17)
    mapping = view.applyCut(np.concatenate([gone, joiners]))
    assert view.n == n - 3000 + nj
    order = np.argsort(mapping[mapping >= 0])
    kept = np.nonzero(mapping >= 0)[0][order]                              # old ids in new-id order
    hb, off, prt = W.packed_endpoints(0, n + nj)
    fresh = rb.MembershipView(K, [hb[off[i]: off[i + 1]].tobytes() for i in kept], prt[kept])
    assert (fresh.getRing(3) == view.getRing(3)).all()
    a, b = view.overlaySpectrum(), fresh.overlaySpectrum()
    assert a[:4] == b[:4]
    assert a.residual <= 1e-3 * 2 * K
    within(a, R.overlay_lambdas(rings_of(view)), K)


def test_a_million_nodes(rb):
    K = 10
    small, big = make_view(rb, 100_000, K).overlaySpectrum(), make_view(rb, 1_000_000, K).overlaySpectrum()
    for sp in (small, big):
        assert sp.residual <= 1e-3 * 2 * K and sp.steps <= 256, sp
        assert 0.40 < sp.ratio < 0.50, sp                                 # the random-regular edge is 2 sqrt(2K - 1) / 2K = 0.436
    assert abs(big.ratio - small.ratio) <= big.residual / (2 * K) + 2e-3, (small, big)


def test_refusals_change_nothing(rb):
    from rapid_b200 import _native as N
    K = 10
    for n in (1, 2):
        with pytest.raises(rb.RapidError) as e:
            make_view(rb, n, K).overlaySpectrum()
        assert e.value.code == N.EINVAL
    view = make_view(rb, 200, K)
    hi, lo = W.node_ids(0, 200)
    view.setNodeIds(hi, lo)
    before = view.overlaySpectrum()
    ring0, cfg = view.getRing(0).copy(), view.currentConfigurationId()
    for kw in ({"tol": 0.0}, {"tol": -1.0}, {"tol": float("nan")}, {"max_steps": 1}, {"max_steps": 513}):
        with pytest.raises(rb.RapidError) as e:
            view.overlaySpectrum(**kw)
        assert e.value.code == N.EINVAL
    assert (view.getRing(0) == ring0).all() and view.currentConfigurationId() == cfg
    assert view.overlaySpectrum()[:4] == before[:4]
    # registered joiners are not part of the graph
    view.registerJoiners(*W.endpoints(200, 5))
    assert view.overlaySpectrum()[:4] == before[:4]


def _quarter_fails(rb, quality):
    n, seed = 50, 3
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed, overlay_quality=quality)
    import random
    for t in sorted(random.Random(seed).sample(range(n), 12)):
        s.setFlags(t, CRASHED)
    assert s.run(30)["converged"]
    return s


def _leave_rejoin_wave(rb, quality):
    n, seed = 30, 34
    s = rb.ClusterSimulation(W.packed_endpoints(0, n), W.node_ids(0, n), seed=seed, overlay_quality=quality)
    gone = [4, 9, 17, 22, 28]
    s.leave(gone)
    assert s.run(40)["converged"]
    for j, t in enumerate(gone):
        hi, lo = W.node_ids((1 << 40) + j, 1)
        s.rejoin(t, int(hi[0]), int(lo[0]))
    assert s.run(40)["converged"] and sorted(s.members()) == list(range(n))
    return s


TIMINGS = ("detect_ms", "classic_ms", "view_change_ms", "handles_ms", "device_ms")


@pytest.mark.parametrize("scenario", [_quarter_fails, _leave_rejoin_wave])
def test_cluster_simulation_reports_the_overlay_of_every_configuration(rb, scenario):
    off, on = scenario(rb, False), scenario(rb, True)
    assert off.initial_overlay is None and len(on.history) == len(off.history) >= 1
    assert all("overlay_ratio" not in h for h in off.history)
    hb, offs, ports = W.packed_endpoints(0, 50)
    K = on.K

    def figure(members):
        v = rb.MembershipView(K, [hb[offs[t]: offs[t + 1]].tobytes() for t in members], ports[list(members)])
        sp = v.overlaySpectrum()
        return sp.ratio, sp.residual

    assert on.initial_overlay == figure(range(on.history[0]["size_before"]))   # members 0..n-1 in id order: the same view, bit for bit
    for a, b in zip(off.history, on.history):
        assert {k: v for k, v in b.items() if k not in TIMINGS + ("overlay_ratio", "overlay_residual")} == \
               {k: v for k, v in a.items() if k not in TIMINGS}
        ratio, res = figure(b["members"])                                 # same members, ids possibly in another order
        assert abs(b["overlay_ratio"] - ratio) <= (b["overlay_residual"] + res) / (2 * K) + 1e-12
        assert 0 < b["overlay_ratio"] < 1 and b["overlay_residual"] <= 1e-3 * 2 * K
    assert len(on.intervals) == len(off.intervals)
    for a, b in zip(off.intervals, on.intervals):
        assert {k: v for k, v in a.items() if k not in ("device_ms", "host_ms")} == {k: v for k, v in b.items() if k not in ("device_ms", "host_ms")}
