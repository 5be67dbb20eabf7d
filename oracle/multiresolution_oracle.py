"""Float64 NumPy restatement of graph_multiresolution's set-up (pygsp/reduction.py:196-382) and of
the effective resistances of graph_sparsify (:84-103), held to tests/golden/multiresolution.npz.

Dense and direct on purpose: it shares no code with the device engine (pygsp_b200/reduction.py,
csrc/schur.cu), whose per-component Schur blocks and Cholesky factor it checks.
"""
import numpy as np
from scipy import sparse

from .pygsp_oracle import laplacian


def largest_eigenvector(L):
    """Eigenvector of the largest eigenvalue of L, times sign(V[0]) (reduction.py:271-277)."""
    L = L.toarray() if sparse.issparse(L) else np.asarray(L)
    _, U = np.linalg.eigh(L)
    V = U[:, -1].copy()
    V *= np.sign(V[0])
    return V


def kron_matrix(M, ind):
    """Dense Schur complement M[ind, ind] - M[ind, comp] M[comp, comp]^-1 M[comp, ind]."""
    M = M.toarray() if sparse.issparse(M) else np.asarray(M, dtype=np.float64)
    ind = np.asarray(ind)
    comp = np.setdiff1d(np.arange(M.shape[0]), ind)
    if comp.size == 0:
        return M[np.ix_(ind, ind)]
    return M[np.ix_(ind, ind)] - M[np.ix_(ind, comp)] @ np.linalg.solve(
        M[np.ix_(comp, comp)], M[np.ix_(comp, ind)])


def kron_graph(W, ind):
    """Adjacency of kron_reduction(Graph(W), ind): -offdiag of the reduced Laplacian (the
    diagonal dropped, as the reference's comment intends; reduction.py:364-372)."""
    Lnew = kron_matrix(laplacian(sparse.csr_matrix(W)), ind)
    Lnew = (Lnew + Lnew.T) / 2
    Wnew = -Lnew
    np.fill_diagonal(Wnew, 0)
    return Wnew


def multiresolution(W, levels, reg_eps=0.005):
    """(Ws, idxs, Kregs) of graph_multiresolution(Graph(W), levels, sparsify=False)."""
    Ws, idxs, Kregs = [np.asarray(sparse.csr_matrix(W).toarray())], [], []
    for _ in range(levels):
        L = laplacian(sparse.csr_matrix(Ws[-1]))
        ind = np.nonzero(largest_eigenvector(L) >= 0)[0]
        Kregs.append(kron_matrix(L + reg_eps * sparse.eye(L.shape[0]), ind))
        Ws.append(kron_graph(Ws[-1], ind))
        idxs.append(ind)
    return Ws, idxs, Kregs


def effective_resistances(W):
    """Dense resistance distances of the graph W from a Cholesky factor of
    L + sum_c 1_c 1_c^T / |c| (one rank-one term per connected component): its inverse is
    L^+ + sum_c 1_c 1_c^T / |c|, and subtracting the added part gives L^+ exactly."""
    from scipy.sparse import csgraph
    W = sparse.csr_matrix(W)
    L = laplacian(W).toarray()
    _, labels = csgraph.connected_components(W, directed=False)
    same = labels[:, None] == labels[None, :]
    sizes = np.bincount(labels)[labels].astype(np.float64)
    added = same / sizes[:, None]
    C = np.linalg.cholesky(L + added)
    Cinv = np.linalg.inv(C)
    pinv = Cinv.T @ Cinv - added
    d = np.diag(pinv)
    return d[:, None] + d[None, :] - pinv - pinv.T
