"""The float64 restatement of NNGraph / ImgPatches / Grid2dImgPatches (oracle/nngraph_oracle.py)
against tests/golden/nngraph.npz (the unmodified PyGSP 0.6.1), without a GPU."""
import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from
from oracle import nngraph_oracle as nno
from pygsp_b200 import utils

DIMS = (1, 3, 8, 27)
METRICS = {"euclidean": 2.0, "manhattan": 1.0, "max_dist": np.inf, "minkowski": 3.0}
SYMS = ("average", "maximum", "fill", "tril", "triu")
SHAPES = {"3x3": (3, 3), "4x2": (4, 2), "5": (5,)}


def assert_csr_equal(got, want, rtol=1e-12):
    got = sparse.csr_matrix(got)
    got.sort_indices()
    np.testing.assert_array_equal(got.indptr, want.indptr)
    np.testing.assert_array_equal(got.indices, want.indices)
    np.testing.assert_allclose(got.data, want.data, rtol=rtol, atol=0)


@pytest.mark.parametrize("nntype", ["knn", "radius"])
@pytest.mark.parametrize("metric", list(METRICS))
@pytest.mark.parametrize("d", DIMS)
def test_nngraph(golden, nntype, metric, d):
    z = golden("nngraph")
    X = z["X_d%d" % d]
    eps = float(z["eps_d%d_%s" % (d, metric)])
    for sym in SYMS:
        tag = "nn_%s_d%d_%s_%s" % (nntype, d, metric, sym)
        W, sigma = nno.nngraph(X, nntype, 10, eps, METRICS[metric], sym)
        assert_csr_equal(W, csr_from(z, tag + "_W"))
        np.testing.assert_allclose(sigma, z[tag + "_sigma"], rtol=1e-13)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("img", ["gray", "rgb"])
def test_patch_graphs(golden, img, shape):
    z = golden("nngraph")
    im = z["img_" + img]
    tag = "%s_%s" % (img, shape)
    np.testing.assert_array_equal(nno.patches(im, SHAPES[shape]), z["ip_%s_X" % tag])
    W, sigma = nno.img_patches(im, SHAPES[shape])
    assert_csr_equal(W, csr_from(z, "ip_%s_W" % tag))
    np.testing.assert_allclose(sigma, z["ip_%s_sigma" % tag], rtol=1e-13)
    W2, _ = nno.grid2d_img_patches(im, SHAPES[shape])
    assert_csr_equal(W2, csr_from(z, "g2ip_%s_W" % tag))


def test_host_symmetrize_fill_matches_reference_docstring():
    """utils.symmetrize(W, 'fill') on the example of pygsp/utils.py:225-228, dense and sparse."""
    W = np.array([[0, 3, 0], [3, 1, 6], [4, 2, 3]], dtype=float)
    want = np.array([[0, 3, 4], [3, 1, 4], [4, 4, 3]], dtype=float)
    np.testing.assert_array_equal(utils.symmetrize(W, "fill"), want)
    np.testing.assert_array_equal(utils.symmetrize(sparse.csr_matrix(W), "fill").toarray(), want)
    np.testing.assert_array_equal(nno.symmetrize(sparse.csr_matrix(W), "fill").toarray(), want)
