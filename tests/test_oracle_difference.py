"""The differential-operator oracle (oracle/difference_oracle.py) against
tests/golden/difference.npz, the output of the unmodified PyGSP 0.6.1 -- no GPU needed."""
import numpy as np
import pytest

from conftest import csr_from, load_golden
from oracle import difference_oracle as do
from oracle import pygsp_oracle as orc

GRAPHS = [str(g) for g in load_golden("difference")["graphs"]]
LAP_TYPES = ("combinatorial", "normalized")


@pytest.mark.parametrize("name", GRAPHS)
def test_edge_list(golden, name):
    z = golden("difference")
    W = csr_from(z, name + "_W")
    directed = orc.is_directed(W)
    assert directed == bool(z[name + "_directed"])
    assert orc.count_edges(W, directed) == int(z[name + "_n_edges"])
    s, t, w = do.edge_list(W, directed)
    np.testing.assert_array_equal(s, z[name + "_sources"])
    np.testing.assert_array_equal(t, z[name + "_targets"])
    np.testing.assert_array_equal(w, z[name + "_weights"])


@pytest.mark.parametrize("lap_type", LAP_TYPES)
@pytest.mark.parametrize("name", GRAPHS)
def test_operator_and_products(golden, name, lap_type):
    z = golden("difference")
    p = "%s_%s_" % (name, lap_type)
    W = csr_from(z, name + "_W")
    D = do.differential_operator(W, lap_type)
    np.testing.assert_array_equal(D.indptr, z[p + "D_indptr"])
    np.testing.assert_array_equal(D.indices, z[p + "D_indices"])
    np.testing.assert_allclose(D.data, z[p + "D_data"], rtol=1e-15, atol=0)
    for key, got in (("grad_x", do.grad(D, z[name + "_x"])), ("grad_X", do.grad(D, z[name + "_X"])),
                     ("div_y", do.div(D, z[name + "_y"])), ("div_Y", do.div(D, z[name + "_Y"]))):
        ref = z[p + key]
        assert got.shape == ref.shape
        np.testing.assert_allclose(got, ref, rtol=0, atol=1e-13 * max(np.abs(ref).max(initial=0), 1))
    L = orc.laplacian(W, lap_type)
    e, E = do.dirichlet_energy(L, z[name + "_x"]), do.dirichlet_energy(L, z[name + "_X"])
    assert np.ndim(e) == 0 and E.shape == (3, 3)
    assert e == pytest.approx(float(z[p + "energy_x"]), rel=1e-12, abs=1e-12)
    np.testing.assert_allclose(E, z[p + "energy_X"], rtol=1e-12, atol=1e-12)
    # L = D D^T, with L the Laplacian of the (symmetrised) graph
    assert abs(D @ D.T - L).max() <= 1e-12 * max(abs(L).max(), 1)


def test_div_checks_the_first_dimension(golden):
    z = golden("difference")
    D = do.differential_operator(csr_from(z, "path4_W"))
    with pytest.raises(ValueError, match="G.Ne = 3"):
        do.div(D, np.ones(4))


def test_doctest_values(golden):
    """difference.py:94-130, 216-322 and graph.py:680-698, 997-1015."""
    z = golden("difference")

    def op(name, lap="combinatorial"):
        return do.differential_operator(csr_from(z, name + "_W"), lap)

    np.testing.assert_allclose(op("tri_undirected").toarray(),
                               [[-1.41421356, 0], [1.41421356, -1], [0, 1]], atol=1e-8)
    np.testing.assert_allclose(op("tri_undirected", "normalized").toarray(),
                               [[-1, 0], [0.81649658, -0.57735027], [0, 1]], atol=1e-8)
    np.testing.assert_allclose(op("tri_directed").toarray(),
                               [[-1, 1, 0], [1, -1, -0.70710678], [0, 0, 0.70710678]], atol=1e-8)
    np.testing.assert_allclose(op("tri_directed", "normalized").toarray(),
                               [[-0.70710678, 0.70710678, 0], [0.63245553, -0.63245553, -0.4472136],
                                [0, 0, 1]], atol=1e-8)
    r2 = np.sqrt(2)
    grads = {("path4", "combinatorial"): [2, 2, -2],
             ("path4_directed", "combinatorial"): [r2, r2, -r2],
             ("path4", "normalized"): [r2, r2, -0.82842712],
             ("path4_directed", "normalized"): [r2, r2, -0.82842712]}
    divs = {("path4", "combinatorial"): [-2, 4, -2, 0],
            ("path4_directed", "combinatorial"): [-r2, 2 * r2, -r2, 0],
            ("path4", "normalized"): [-2, 2 * r2, -r2, 0],
            ("path4_directed", "normalized"): [-2, 2 * r2, -r2, 0]}
    for (name, lap), want in grads.items():
        D = op(name, lap)
        np.testing.assert_allclose(do.grad(D, [0, 2, 4, 2]), want, atol=1e-8)
        np.testing.assert_allclose(do.div(D, [2, -2, 0]), divs[name, lap], atol=1e-8)
    for name, energy, grad in (("path5", 8.0, [2, 0, 2, 0]),
                               ("path5_directed", 4.0, [r2, 0, r2, 0])):
        W = csr_from(z, name + "_W")
        assert do.dirichlet_energy(orc.laplacian(W), [0, 2, 2, 4, 4]) == energy
        np.testing.assert_allclose(do.grad(op(name), [0, 2, 2, 4, 4]), grad, atol=1e-8)
    s, t, w = do.edge_list(csr_from(z, "edges_directed_W"), True)
    assert (list(s), list(t), list(w)) == ([0, 1, 1], [1, 0, 2], [3, 3, 4])
    s, t, w = do.edge_list(csr_from(z, "edges_undirected_W"), False)
    assert (list(s), list(t), list(w)) == ([0, 1], [1, 2], [3, 4])
