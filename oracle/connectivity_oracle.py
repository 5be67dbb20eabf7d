"""CPU oracle for the connectivity methods of PyGSP 0.6.1 (pygsp/graphs/graph.py:192-508).

TEST INFRASTRUCTURE ONLY, like ``oracle/pygsp_oracle.py`` beside it.  A NumPy / SciPy
restatement of ``is_connected``, ``is_weighted``, ``extract_components`` and ``subgraph`` that
``tests/test_oracle_connectivity.py`` holds to ``tests/golden/connectivity.npz``, the output of
the unmodified reference.  Connectivity comes from ``scipy.sparse.csgraph``.
"""
import numpy as np
from scipy import sparse
from scipy.sparse import csgraph

from . import pygsp_oracle as orc


def is_connected(W):
    """graph.py:340-366: every vertex reachable from 0 (through W and W^T if directed); an edge
    is any stored entry.  N = 0 raises IndexError."""
    W = sparse.csr_matrix(W)
    if W.shape[0] == 0:
        raise IndexError("index 0 is out of bounds for axis 0 with size 0")
    A = sparse.csr_matrix((np.ones(W.nnz), W.indices, W.indptr), shape=W.shape)
    directed = orc.is_directed(W)
    n, _ = csgraph.connected_components(A, directed=directed, connection="strong")
    return n == 1


def is_weighted(W):
    """graph.py:292: not all(W.data == 1)."""
    return not np.all(sparse.csr_matrix(W).data == 1)


def component_labels(W):
    """Labels of the components of A = W > 0 (graph.py:480-500): the smallest vertex id of each
    vertex's component."""
    W = sparse.csr_matrix(W)
    _, labels = csgraph.connected_components(W > 0, directed=False)
    first = np.full(labels.max(initial=-1) + 1, W.shape[0])
    np.minimum.at(first, labels, np.arange(W.shape[0]))
    return first[labels]


def subgraph(W, vertices):
    """W[vertices, :][:, vertices] (graph.py:247) as canonical CSR."""
    S = sparse.csr_matrix(W)[vertices, :][:, vertices].tocsr()
    S.sum_duplicates()
    S.sort_indices()
    return S


def extract_components(W):
    """[(orig_idx, W of the component)] in order of smallest vertex (graph.py:444-508)."""
    W = sparse.csr_matrix(W)
    if orc.is_directed(W):
        raise NotImplementedError("Directed graphs not supported yet.")
    labels = component_labels(W)
    out = []
    for root in np.unique(labels):
        ids = np.flatnonzero(labels == root).astype(np.int64)
        out.append((ids, subgraph(W, ids)))
    return out
