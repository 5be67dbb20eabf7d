"""Tree multiresolution rules on the host (oracle/tree_oracle.py): a hand-worked weighted tree with
its levels written out for every reduction method, and the Euler-tour rooting of the device
(restated in NumPy) against BFS depths and parents on seeded random trees, paths and stars."""
import numpy as np
import pytest
from scipy import sparse

from oracle import tree_oracle as tro


def _tree(n, edges):
    u, v, w = (np.array(x) for x in zip(*edges))
    return sparse.csr_matrix((np.concatenate([w, w]).astype(np.float64),
                              (np.concatenate([u, v]), np.concatenate([v, u]))), shape=(n, n))


# Root 1.  Depths: 1:0; 0, 5:1; 2, 6:2; 3:3; 4:4.
SEVEN = _tree(7, [(1, 0, 2.0), (0, 2, 4.0), (2, 3, 1.0), (3, 4, 2.0), (1, 5, 8.0), (5, 6, 4.0)])


def _dense_edges(W):
    W = sparse.csr_matrix(W)
    return {(int(i), int(j)): float(x) for i, j, x in zip(*sparse.find(sparse.triu(W)))}


@pytest.mark.parametrize("method", tro.METHODS)
def test_seven_vertex_tree_by_hand(method):
    levels = tro.tree_multiresolution_levels(SEVEN, 4, method, root=1)
    # level 1 keeps 1, 2, 4, 6 (new ids 0..3): 2 -> 1 through 0, 4 -> 2 through 3, 6 -> 1 through 5
    np.testing.assert_array_equal(levels[0]["keep"], [1, 2, 4, 6])
    assert levels[0]["root"] == 0
    np.testing.assert_array_equal(levels[0]["depth"], [0, 1, 2, 1])
    np.testing.assert_array_equal(levels[0]["parent"], [0, 0, 1, 0])
    # level 2 keeps new ids 0 and 2 (vertices 1 and 4): 4 -> 1 through 2
    np.testing.assert_array_equal(levels[1]["keep"], [0, 2])
    np.testing.assert_array_equal(levels[1]["orig_idx"], [1, 4])
    # then one vertex, repeated
    np.testing.assert_array_equal(levels[2]["keep"], [0])
    np.testing.assert_array_equal(levels[3]["keep"], [0])
    for lev in levels[2:]:
        assert lev["W"].shape == (1, 1) and lev["W"].nnz == 0 and lev["root"] == 0
        np.testing.assert_array_equal(lev["orig_idx"], [1])
    if method == "unweighted":
        l1 = {(0, 1): 1.0, (1, 2): 1.0, (0, 3): 1.0}
        l2 = {(0, 1): 1.0}
    elif method == "sum":
        l1 = {(0, 1): 4.0 + 2.0, (1, 2): 2.0 + 1.0, (0, 3): 4.0 + 8.0}
        l2 = {(0, 1): (2.0 + 1.0) + (4.0 + 2.0)}
    else:
        r = [1.0 / (1.0 / 4.0 + 1.0 / 2.0), 1.0 / (1.0 / 2.0 + 1.0 / 1.0),
             1.0 / (1.0 / 4.0 + 1.0 / 8.0)]
        l1 = {(0, 1): r[0], (1, 2): r[1], (0, 3): r[2]}
        l2 = {(0, 1): 1.0 / (1.0 / r[1] + 1.0 / r[0])}
        assert l2[(0, 1)] == pytest.approx(4.0 / 9.0, rel=1e-15)
    assert _dense_edges(levels[0]["W"]) == l1
    assert _dense_edges(levels[1]["W"]) == l2
    for lev in levels:
        W = lev["W"]
        assert (W != W.T).nnz == 0 and W.diagonal().sum() == 0
        assert W.nnz == 2 * (W.shape[0] - 1)


def test_float32_rounds_once_per_level():
    levels = tro.tree_multiresolution_levels(SEVEN, 2, "resistance_distance", root=1,
                                             dtype=np.float32)
    r1 = np.float32(1.0 / (1.0 / 2.0 + 1.0 / 1.0))
    r0 = np.float32(1.0 / (1.0 / 4.0 + 1.0 / 2.0))
    assert levels[0]["W"].dtype == np.float32
    assert levels[1]["W"][0, 1] == np.float32(1.0 / (1.0 / float(r1) + 1.0 / float(r0)))


def test_directed_support_and_loops():
    # a directed path with a self-loop: the support is the tree, one-way edges weigh 1/2
    W = sparse.csr_matrix((np.ones(4), ([0, 1, 2, 2], [1, 2, 3, 2])), shape=(4, 4))
    Ws = (W + W.T) / 2
    levels = tro.tree_multiresolution_levels(Ws, 1, "sum", root=0)
    np.testing.assert_array_equal(levels[0]["keep"], [0, 2])
    assert _dense_edges(levels[0]["W"]) == {(0, 1): 1.0}


def test_coords_follow_the_kept_vertices():
    coords = np.arange(14.0).reshape(7, 2)
    levels = tro.tree_multiresolution_levels(SEVEN, 2, "sum", root=1, coords=coords)
    np.testing.assert_array_equal(levels[0]["coords"], coords[[1, 2, 4, 6]])
    np.testing.assert_array_equal(levels[1]["coords"], coords[[1, 4]])


def _trees():
    rng = np.random.default_rng(2024)
    for t in range(200):
        kind = t % 4
        n = int(rng.integers(1, 300))
        if kind == 0:                                       # random recursive, relabelled
            W = tro.random_tree(n, seed=t)
        elif kind == 1:                                     # path, relabelled
            p = rng.permutation(n)
            W = _tree(n, [(p[i], p[i + 1], 1.0 + i) for i in range(n - 1)]) if n > 1 \
                else sparse.csr_matrix((1, 1))
        elif kind == 2:                                     # star about a random centre
            c = int(rng.integers(n))
            W = _tree(n, [(c, v, 2.0) for v in range(n) if v != c]) if n > 1 \
                else sparse.csr_matrix((1, 1))
        else:                                               # random recursive, not relabelled
            W = tro.random_tree(n, seed=t, relabel=False)
        yield W, int(rng.integers(n))


def test_euler_tour_equals_bfs():
    count = 0
    for W, root in _trees():
        Ws = tro.symmetric_support(W)
        d_bfs, p_bfs, w_bfs = tro.bfs_depths(Ws, root)
        d_tour, p_tour, w_tour = tro.euler_tour_depths(Ws, root)
        np.testing.assert_array_equal(d_tour, d_bfs)
        np.testing.assert_array_equal(p_tour, p_bfs)
        np.testing.assert_array_equal(w_tour, w_bfs)
        count += 1
    assert count == 200


def test_euler_tour_refuses_a_cycle():
    ring = _tree(4, [(0, 1, 1.0), (1, 2, 1.0), (2, 3, 1.0), (3, 0, 1.0)])
    with pytest.raises(ValueError):
        tro.euler_tour_depths(ring, 0)


def test_unknown_method():
    with pytest.raises(ValueError, match="Unknown graph reduction method"):
        tro.tree_multiresolution_levels(SEVEN, 1, "kron", root=1)
