"""Dense NumPy / SciPy restatement of the effective-resistance sketch of
``graph_sparsify(resistances='sketch')`` (pygsp_b200/reduction.py ``_edge_resistances``,
csrc/resistance.cu).

Test infrastructure: nothing under pygsp_b200/ imports this module.

The reference computes ``resistance_distances[start_nodes, end_nodes]`` from a dense inverse
(pygsp/reduction.py:84, :101).  The sketch replaces it by Spielman-Srivastava's estimator
R~_e = ||Z (chi_u - chi_v)||^2, Z = Q W^1/2 B L^+ / sqrt(k), with the same +-1 signs Q as the
device (``random_graphs_oracle.curand4``): the sign of edge {a < b} in column j is +1 when bit
(j mod 128) of the 128 bits of curand4(key, a N + b, j div 128) is 0, else -1, bit t being bit
(t mod 32) of word (t div 32) of (x, y, z, w).  B has +1 at an edge's larger end.

* ``sketch_rhs``         -- the block Y = D^-1/2 B^T W^1/2 Q^T / sqrt(k) of columns j0 .. j0+width-1.
* ``sketch_resistances`` -- R~ of the edges, with L^+ from a dense ``pinv`` in place of CG, so a
  comparison with the device does not depend on the JL randomness.
"""
import numpy as np
from scipy import sparse

from oracle.random_graphs_oracle import curand4


def _edges(W):
    """(a, b, w) of the edges a < b of the symmetric matrix W, in row-major order of the upper
    triangle."""
    T = sparse.triu(sparse.csr_matrix(W, dtype=np.float64), k=1).tocsr()
    T.eliminate_zeros()
    T = T.tocoo()
    return T.row.astype(np.int64), T.col.astype(np.int64), T.data


def signs(a, b, n, key, j0, width):
    """(ne, width) +-1 signs of the edges {a[e] < b[e]} in columns j0 .. j0 + width - 1."""
    j = np.arange(j0, j0 + width, dtype=np.int64)
    sub = (a * n + b).astype(np.uint64)
    t = np.unique(j >> 7)
    words = np.stack(curand4(key, sub[:, None], t[None, :].astype(np.uint64)))  # (4, ne, len(t))
    word = words[(j >> 5) & 3, :, np.searchsorted(t, j >> 7)].T                 # (ne, width)
    bit = (word >> (j & 31).astype(np.uint64)) & np.uint64(1)
    return 1.0 - 2.0 * bit.astype(np.float64)


def _dinv(W):
    d = np.asarray(sparse.csr_matrix(W).sum(axis=1)).ravel()
    return np.where(d > 0, 1.0 / np.sqrt(np.where(d > 0, d, 1.0)), 0.0)


def sketch_rhs(W, key, k, j0, width):
    """Columns j0 .. j0 + width - 1 of D^-1/2 B^T W^1/2 Q^T / sqrt(k), an (N, width) array."""
    n = W.shape[0]
    a, b, w = _edges(W)
    S = signs(a, b, n, key, j0, width) * np.sqrt(w)[:, None]
    Y = np.zeros((n, width))
    np.add.at(Y, b, S)           # +1 at the larger end
    np.add.at(Y, a, -S)
    return _dinv(W)[:, None] * Y / np.sqrt(k)


def sketch_resistances(W, key, k, block=256):
    """(start, end, R~) over the edges start > end of W in row-major order of the lower triangle
    (the order of graph_sparsify's edges), with Z from the dense pseudo-inverse of the
    Jacobi-scaled Laplacian."""
    W = sparse.csr_matrix(W, dtype=np.float64)
    n = W.shape[0]
    dinv = _dinv(W)
    L = sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W
    Lhat = dinv[:, None] * L.toarray() * dinv[None, :]
    P = np.linalg.pinv(Lhat, hermitian=True)
    T = sparse.tril(W, k=-1).tocsr()
    T.eliminate_zeros()
    T = T.tocoo()
    start, end = T.row.astype(np.int64), T.col.astype(np.int64)
    R = np.zeros(start.size)
    for j0 in range(0, k, block):
        wb = min(block, k - j0)
        Z = dinv[:, None] * (P @ sketch_rhs(W, key, k, j0, wb))
        R += ((Z[start] - Z[end]) ** 2).sum(axis=1)
    return start, end, R


def pinv_resistances(W):
    """(start, end, R) exact effective resistances of the same edges from pinv(L)."""
    W = sparse.csr_matrix(W, dtype=np.float64)
    L = (sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W).toarray()
    P = np.linalg.pinv(L, hermitian=True)
    T = sparse.tril(W, k=-1).tocsr()
    T.eliminate_zeros()
    T = T.tocoo()
    start, end = T.row.astype(np.int64), T.col.astype(np.int64)
    d = np.diag(P)
    return start, end, d[start] + d[end] - 2 * P[start, end]


def two_component_graph(seed=0):
    """A weighted symmetric adjacency (SciPy CSR, 13 vertices) with three components: a random
    connected graph on 0..6, a ring with a chord on 7..11 (weights over three decades) and the
    isolated vertex 12."""
    rng = np.random.default_rng(seed)
    rows, cols = list(range(6)), list(range(1, 7))          # a path keeps 0..6 connected
    for a, b in ((0, 3), (1, 5), (2, 6), (0, 6), (3, 5)):
        rows.append(a)
        cols.append(b)
    ring = [7, 8, 9, 10, 11]
    for p in range(5):
        rows.append(ring[p])
        cols.append(ring[(p + 1) % 5])
    rows.append(7)
    cols.append(9)
    w = 10.0 ** rng.uniform(-1.5, 1.5, len(rows))
    W = sparse.coo_matrix((w, (rows, cols)), shape=(13, 13))
    return (W + W.T).tocsr()
