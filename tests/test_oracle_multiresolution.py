"""The float64 restatement of graph_multiresolution's set-up (oracle/multiresolution_oracle.py)
against tests/golden/multiresolution.npz (the unmodified PyGSP 0.6.1), without a GPU."""
import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from
from oracle import multiresolution_oracle as mro
from oracle.pygsp_oracle import laplacian

CASES = ["s256", "s1000", "grid"]


def _rowwise(got, want):
    """max over rows of max|got - want| / max|want| (the row's largest weight)."""
    got, want = np.asarray(got), np.asarray(want)
    scale = np.maximum(np.abs(want).max(axis=1), 1e-300)
    return float((np.abs(got - want).max(axis=1) / scale).max())


@pytest.mark.parametrize("name", CASES)
def test_kron_both_branches(golden, name):
    z = golden("multiresolution")
    W = csr_from(z, name + "_W")
    ind = z[name + "_ind"]
    got_w = mro.kron_graph(W, ind)
    assert _rowwise(got_w, csr_from(z, name + "_kronW").toarray()) <= 1e-10
    L = laplacian(W)
    got_k = mro.kron_matrix(L + 0.005 * sparse.eye(W.shape[0]), ind)
    assert _rowwise(got_k, csr_from(z, name + "_kreg").toarray()) <= 1e-10


@pytest.mark.parametrize("name", ["s256", "grid"])
def test_largest_eigenvector_split(golden, name):
    z = golden("multiresolution")
    V = mro.largest_eigenvector(laplacian(csr_from(z, name + "_W")))
    np.testing.assert_allclose(V, z[name + "_V"], atol=1e-10)
    np.testing.assert_array_equal(np.nonzero(V >= 0)[0], z[name + "_ind"])
    assert int(z[name + "_ambiguous"]) == 0


def test_multiresolution_levels(golden):
    z = golden("multiresolution")
    levels = int(z["mr_levels"])
    Ws, idxs, Kregs = mro.multiresolution(csr_from(z, "mr_W0"), levels)
    for i in range(levels):
        np.testing.assert_array_equal(idxs[i], z["mr_idx%d" % (i + 1)])
        assert _rowwise(Ws[i + 1], csr_from(z, "mr_W%d" % (i + 1)).toarray()) <= 1e-10
        assert _rowwise(Kregs[i], csr_from(z, "mr_Kreg%d" % i).toarray()) <= 1e-10


def test_pyramid_fixture_split_is_well_defined(golden):
    """The levels of tests/golden/pyramid.npz: the smallest |V_i| is 2e-11 max|V| (level 1), far
    above the round-off of a dense float64 eigensolver, so a float64 eigenvector reproduces
    idx1..3 exactly."""
    z = golden("pyramid")
    for i in range(int(z["levels"])):
        V = mro.largest_eigenvector(laplacian(csr_from(z, "W%d" % i)))
        assert np.abs(V).min() > 1e-11 * np.abs(V).max()
        np.testing.assert_array_equal(np.nonzero(V >= 0)[0], z["idx%d" % (i + 1)])


def test_effective_resistances_match_pinv():
    A = sparse.random(60, 60, density=0.08, random_state=7)
    A = A + A.T
    A.setdiag(0)
    A.eliminate_zeros()
    # a second component and an isolated vertex
    B = sparse.block_diag([A, sparse.csr_matrix(np.array([[0, 2.0], [2.0, 0]])),
                           sparse.csr_matrix((1, 1))]).tocsr()
    for W in (A, B):
        L = laplacian(sparse.csr_matrix(W)).toarray()
        P = np.linalg.pinv(L)
        d = np.diag(P)
        want = d[:, None] + d[None, :] - 2 * P
        got = mro.effective_resistances(W)
        assert np.abs(got - want).max() <= 1e-9 * np.abs(want).max()
