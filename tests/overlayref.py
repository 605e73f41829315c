"""Plain reference of the monitoring overlay's spectrum (DESIGN.md §4.13), for the tests of rapid_view_overlay_spectrum: the
observer graph of a view as a scipy sparse matrix built from its rings, its extreme eigenvalues below the trivial 2K from
scipy's solvers, and the first Lanczos steps from the documented seeded start vector.  NOT a pytest module."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

DENSE_LIMIT = 2000


def overlay_matrix(rings):
    """rings: K sequences of the n member ids in ring order -> A = sum_k (P_k + P_k^T) as CSR, P_k = successor on ring k;
    an edge present on m rings has weight m (duplicates are summed)"""
    rings = [np.asarray(r, np.int64) for r in rings]
    n = len(rings[0])
    rows = np.concatenate([r for r in rings])
    cols = np.concatenate([np.roll(r, -1) for r in rings])
    P = sp.coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(n, n)).tocsr()
    return (P + P.T).tocsr()


def matrix_from_tables(obs, subj):
    """the same graph from per-node observer and subject lists: A[v][obs[v][k]] += 1, A[v][subj[v][k]] += 1"""
    obs, subj = np.asarray(obs, np.int64), np.asarray(subj, np.int64)
    n, K = obs.shape
    rows = np.repeat(np.arange(n), 2 * K)
    cols = np.concatenate([obs, subj], axis=1).ravel()
    return sp.coo_matrix((np.ones(len(rows)), (rows, cols)), shape=(n, n)).tocsr()


def _dense_lambdas(A):
    w = np.linalg.eigvalsh(A.toarray())
    return float(w[-2]), float(w[0])                  # the top one is 2K (all-ones vector)


def _sparse_lambdas(A, K):
    """A - (2K / n) 1 1^T moves the trivial eigenvalue to 0, inside the spectrum's hull, and leaves the complement alone"""
    n = A.shape[0]
    ones = np.ones(n) / np.sqrt(n)
    op = spla.LinearOperator((n, n), matvec=lambda x: A @ x - (2.0 * K) * ones * (ones @ x), dtype=np.float64)
    v0 = np.random.default_rng(1).standard_normal(n)
    hi = spla.eigsh(op, k=1, which="LA", tol=1e-8, v0=v0, ncv=min(n - 1, 64), maxiter=20000, return_eigenvectors=False)
    lo = spla.eigsh(op, k=1, which="SA", tol=1e-8, v0=v0, ncv=min(n - 1, 64), maxiter=20000, return_eigenvectors=False)
    return float(hi[0]), float(lo[0])


def overlay_lambdas(rings, dense=None):
    """(lambda2, lambda_min) of the overlay restricted to the complement of the all-ones vector; dense eigvalsh up to
    DENSE_LIMIT nodes, eigsh beyond (dense=True / False forces one)"""
    A = overlay_matrix(rings)
    if dense is None:
        dense = A.shape[0] <= DENSE_LIMIT
    return _dense_lambdas(A) if dense else _sparse_lambdas(A, len(rings))


def splitmix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        z = x + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def start_vector(n, seed):
    """x[v] = 2 u - 1, u = (splitmix64(seed + v) >> 11) * 2^-53; mean removed; normalised"""
    with np.errstate(over="ignore"):
        h = splitmix64(np.uint64(seed & 0xFFFFFFFFFFFFFFFF) + np.arange(n, dtype=np.uint64))
    x = 2.0 * ((h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53) - 1.0
    x -= x.mean()
    return x / np.linalg.norm(x)


def lanczos(A, seed, steps):
    """alpha[steps], beta[steps] of Lanczos on A in the complement of the all-ones vector from start_vector(n, seed), every
    new vector orthogonalised against all earlier ones"""
    n = A.shape[0]
    V = [start_vector(n, seed)]
    alpha, beta = [], []
    for j in range(steps):
        w = A @ V[j]
        alpha.append(float(w @ V[j]))
        w = w - w.mean() - alpha[j] * V[j] - (beta[j - 1] * V[j - 1] if j else 0.0)
        for u in V:
            w = w - (u @ w) * u
        beta.append(float(np.linalg.norm(w)))
        V.append(w / beta[j])
    return np.array(alpha), np.array(beta)


def ritz_ends(alpha, beta):
    """(largest, smallest) eigenvalue of tridiag(beta[:-1], alpha, beta[:-1]) and the larger |beta[-1] * last eigenvector
    component| of the two"""
    m = len(alpha)
    T = np.diag(alpha) + np.diag(beta[: m - 1], 1) + np.diag(beta[: m - 1], -1)
    w, S = np.linalg.eigh(T)
    return float(w[-1]), float(w[0]), float(abs(beta[m - 1]) * max(abs(S[-1, -1]), abs(S[-1, 0])))
