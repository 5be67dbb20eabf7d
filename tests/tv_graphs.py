"""Seeded adjacency matrices for the total-variation prox tests (CPU and GPU)."""
import numpy as np
from scipy import sparse
from scipy.sparse import csgraph


def path(n):
    """Path graph with unit weights (no graphs.Path here): W = diags."""
    return sparse.diags([np.ones(n - 1), np.ones(n - 1)], [-1, 1], format="csr")


def geometric(n=60, seed=0, radius2=0.06):
    """Weighted geometric graph: Gaussian weights between points closer than sqrt(radius2)."""
    pts = np.random.default_rng(seed).uniform(size=(n, 2))
    d2 = ((pts[:, None] - pts[None]) ** 2).sum(-1)
    return sparse.csr_matrix(np.where((d2 < radius2) & (d2 > 0), np.exp(-d2 / 0.02), 0.0))


def six_decades(n=80, seed=1):
    """Geometric structure, weights spread log-uniformly over 1e-3 .. 1e3."""
    W = sparse.triu(geometric(n, seed), k=1).tocoo()
    w = 10.0 ** np.random.default_rng(seed).uniform(-3, 3, W.nnz)
    U = sparse.csr_matrix((w, (W.row, W.col)), shape=W.shape)
    return (U + U.T).tocsr()


def directed(n=50, seed=2):
    W = sparse.triu(sparse.random(n, n, density=0.1, random_state=seed), k=1).tocsr()
    W.data += 0.1
    return W


def disconnected(seed=3):
    return sparse.block_diag([geometric(30, seed), path(12), geometric(20, seed + 1)]).tocsr()


def with_loops(n=40, seed=4):
    W = geometric(n, seed).tolil()
    for i in range(0, n, 3):
        W[i, i] = 0.5 + i / n
    return W.tocsr()


def grid(rows=6, cols=7):
    idx = np.arange(rows * cols).reshape(rows, cols)
    r = np.r_[idx[:, :-1].ravel(), idx[:-1, :].ravel()]
    c = np.r_[idx[:, 1:].ravel(), idx[1:, :].ravel()]
    U = sparse.csr_matrix((np.ones(r.size), (r, c)), shape=(rows * cols,) * 2)
    return (U + U.T).tocsr()


def lmax_of(D):
    """Largest eigenvalue of D D^T (dense)."""
    return float(np.linalg.eigvalsh((D @ D.T).toarray()).max())


def component_means(W, x):
    n_comp, labels = csgraph.connected_components(W, directed=False)
    X = np.asarray(x, dtype=np.float64).reshape(W.shape[0], -1)
    out = np.empty_like(X)
    for c in range(n_comp):
        out[labels == c] = X[labels == c].mean(axis=0)
    return out


def mean_bound(W, D, x):
    """||u0||_inf, u0 = D^T L^+ (x - component means): for gamma >= it (combinatorial
    Laplacian) the prox is the component means."""
    L = (D @ D.T).toarray()
    X = np.asarray(x, dtype=np.float64).reshape(W.shape[0], -1)
    u0 = D.T @ (np.linalg.pinv(L) @ (X - component_means(W, X)))
    return float(np.abs(u0).max())
