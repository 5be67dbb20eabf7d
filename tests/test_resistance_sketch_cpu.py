"""The resistance sketch of graph_sparsify(resistances='sketch'), restated in NumPy
(oracle/resistance_sketch_oracle.py), against exact resistances from pinv: the estimator and its
Philox signs are right before the device is compared with them."""
import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import csgraph

from oracle import resistance_sketch_oracle as rso

KEY = 0x0123456789ABCDEF


def ring(n):
    i = np.arange(n)
    W = sparse.coo_matrix((np.ones(n), (i, (i + 1) % n)), shape=(n, n))
    return (W + W.T).tocsr()


def grid2d(n):
    return sparse.kronsum(_path(n), _path(n)).tocsr()


def _path(n):
    i = np.arange(n - 1)
    W = sparse.coo_matrix((np.ones(n - 1), (i, i + 1)), shape=(n, n))
    return (W + W.T).tocsr()


GRAPHS = {"ring16": lambda: ring(16), "grid6": lambda: grid2d(6),
          "two_components": rso.two_component_graph}


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_sketch_matches_pinv(name):
    W = GRAPHS[name]()
    s, e, R = rso.sketch_resistances(W, KEY, 20000)
    s2, e2, Rx = rso.pinv_resistances(W)
    np.testing.assert_array_equal(s, s2)
    np.testing.assert_array_equal(e, e2)
    assert np.abs(R / Rx - 1).max() <= 0.05


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_sketch_columns_sum_to_zero_per_component(name):
    """D^1/2 Y = B^T W^1/2 Q^T / sqrt(k) sums to zero over every component, so the scaled system
    D^-1/2 L D^-1/2 U = Y is consistent."""
    W = GRAPHS[name]()
    ncomp, labels = csgraph.connected_components(W, directed=False)
    d = np.asarray(W.sum(axis=1)).ravel()
    for j0, width in ((0, 256), (256, 44), (8, 8), (120, 256)):
        Y = rso.sketch_rhs(W, KEY, 400, j0, width)
        X = np.sqrt(d)[:, None] * Y
        scale = np.abs(X).max()
        for c in range(ncomp):
            assert np.abs(X[labels == c].sum(axis=0)).max() <= 1e-12 * scale


@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_foster(name):
    """sum_e w_e R~_e is within 1 % of N - #components (Foster's theorem)."""
    W = GRAPHS[name]()
    ncomp, _ = csgraph.connected_components(W, directed=False)
    s, e, R = rso.sketch_resistances(W, KEY, 20000)
    w = np.asarray(W[s, e]).ravel()
    assert abs((w * R).sum() / (W.shape[0] - ncomp) - 1) <= 0.01


def test_default_dim_and_block_width():
    """k = ceil(24 ln N / 0.5^2); the block width depends on N and k only: min(k, 256, w_mem),
    w_mem the largest power of two >= 8 with 5 * 8 * N * w_mem <= 32 GiB."""
    from pygsp_b200 import reduction as red
    assert red._sketch_dim(3000) == 769
    assert red._sketch_dim(10 ** 6) == 1327
    assert red._sketch_dim(1) == 1
    assert red._sketch_width(3000, 769) == 256
    assert red._sketch_width(3000, 44) == 44
    assert red._sketch_width(10 ** 7, 1327) == 64
    n8 = (32 << 30) // (5 * 8 * 8)
    assert red._sketch_width(n8, 1327) == 8
    with pytest.raises(ValueError, match="GB of device memory"):
        red._sketch_width(n8 + 1, 1327)
