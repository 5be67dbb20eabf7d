"""The connectivity oracle (oracle/connectivity_oracle.py) against tests/golden/connectivity.npz,
the output of the unmodified PyGSP 0.6.1 -- no GPU needed."""
import numpy as np
import pytest

from conftest import csr_from, load_golden
from oracle import connectivity_oracle as co
from oracle import pygsp_oracle as orc

GRAPHS = [str(g) for g in load_golden("connectivity")["graphs"]]
SUBGRAPHS = [str(s) for s in load_golden("connectivity")["subgraphs"]]


def _same_csr(got, z, prefix):
    ref = csr_from(z, prefix)
    assert got.shape == ref.shape
    np.testing.assert_array_equal(got.indptr, ref.indptr)
    np.testing.assert_array_equal(got.indices, ref.indices)
    np.testing.assert_array_equal(got.data, ref.data)


@pytest.mark.parametrize("name", GRAPHS)
def test_flags_and_components(golden, name):
    z = golden("connectivity")
    W = csr_from(z, name + "_W")
    assert orc.is_directed(W) == bool(z[name + "_directed"])
    assert co.is_connected(W) == bool(z[name + "_connected"])
    assert co.is_weighted(W) == bool(z[name + "_weighted"])
    if bool(z[name + "_directed"]):
        with pytest.raises(NotImplementedError, match="Directed graphs not supported yet."):
            co.extract_components(W)
        return
    comps = co.extract_components(W)
    assert len(comps) == int(z[name + "_n_components"])
    for k, (ids, C) in enumerate(comps):
        p = "%s_comp%d" % (name, k)
        np.testing.assert_array_equal(ids, z[p + "_orig_idx"])
        _same_csr(C, z, p + "_W")


def test_negative_edge_splits_components(golden):
    z = golden("connectivity")
    W = csr_from(z, "negative_W")
    assert co.is_connected(W)
    assert [list(ids) for ids, _ in co.extract_components(W)] == [[0, 1], [2, 3]]


@pytest.mark.parametrize("case", SUBGRAPHS)
def test_subgraph(golden, case):
    z = golden("connectivity")
    g = str(z[case + "_graph"])
    sel = z[case + "_sel"]
    _same_csr(co.subgraph(csr_from(z, g + "_W"), sel), z, case + "_W")
    np.testing.assert_array_equal(z[g + "_coords"][sel].reshape(-1, 2), z[case + "_coords"])
    np.testing.assert_array_equal(z[g + "_signal"][sel].reshape(-1, 3), z[case + "_signal"])


def test_empty_graph():
    from scipy import sparse
    with pytest.raises(IndexError):
        co.is_connected(sparse.csr_matrix((0, 0)))
    assert co.extract_components(sparse.csr_matrix((0, 0))) == []
