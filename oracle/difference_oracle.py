"""CPU oracle for the graph differential operator of PyGSP 0.6.1 (pygsp/graphs/difference.py).

TEST INFRASTRUCTURE ONLY, like ``oracle/pygsp_oracle.py`` beside it (whose degree and
Laplacian it uses).  A float64 NumPy / SciPy restatement of ``get_edge_list``,
``compute_differential_operator``, ``grad``, ``div`` and ``dirichlet_energy`` that
``tests/test_oracle_difference.py`` holds to ``tests/golden/difference.npz``, the output of
the unmodified reference.
"""
import numpy as np
from scipy import sparse

from . import pygsp_oracle as orc


def edge_list(W, directed):
    """(sources, targets, weights) of graph.py:1019-1029: every stored entry of a directed W,
    the upper triangle (diagonal included) of an undirected one, in row-major order."""
    W = sparse.csr_matrix(W, dtype=np.float64)
    C = W.tocoo() if directed else sparse.triu(W, format="coo")
    order = np.lexsort((C.col, C.row))
    return (C.row[order].astype(np.int32), C.col[order].astype(np.int32),
            C.data[order].astype(np.float64))


def differential_operator(W, lap_type="combinatorial", directed=None):
    """D (N x Ne) as canonical ``csc_matrix`` (difference.py:144-166).

    combinatorial: -sqrt(w) at the source, +sqrt(w) at the target; normalized:
    -sqrt(w / dw[s]) and +sqrt(w / dw[t]); both / sqrt(2) when directed.  A self-loop's two
    entries cancel and ``eliminate_zeros`` (:166) removes them.
    """
    W = sparse.csr_matrix(W, dtype=np.float64)
    if directed is None:
        directed = orc.is_directed(W)
    sources, targets, weights = edge_list(W, directed)
    n = len(sources)
    dw = orc.weighted_degree(W, directed)
    values = np.empty(2 * n)
    if lap_type == "combinatorial":
        values[:n] = -np.sqrt(weights)
        values[n:] = -values[:n]
    elif lap_type == "normalized":
        values[:n] = -np.sqrt(weights / dw[sources])
        values[n:] = +np.sqrt(weights / dw[targets])
    else:
        raise ValueError("Unknown lap_type {}".format(lap_type))
    if directed:
        values /= np.sqrt(2)
    D = sparse.csc_matrix((values, (np.concatenate([sources, targets]),
                                    np.concatenate([np.arange(n), np.arange(n)]))),
                          shape=(W.shape[0], n))
    D.eliminate_zeros()
    return D


def grad(D, x):
    """D^T x (difference.py:243-244)."""
    return D.T.dot(np.asarray(x, dtype=np.float64))


def div(D, y):
    """D y (difference.py:325-331), with its check of the first dimension."""
    y = np.asanyarray(y, dtype=np.float64)
    if y.shape[0] != D.shape[1]:
        raise ValueError("First dimension must be the number of edges "
                         "G.Ne = {}, got {}.".format(D.shape[1], y.shape))
    return D.dot(y)


def dirichlet_energy(L, x):
    """x^T L x (graph.py:701-702): a scalar for a vector, (Nsig, Nsig) for a block."""
    x = np.asarray(x, dtype=np.float64)
    return x.T.dot(L.dot(x))
