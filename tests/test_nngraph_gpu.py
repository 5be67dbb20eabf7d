"""Nearest-neighbour graphs on the device (csrc/neighbors.cu, graphs.NNGraph / ImgPatches /
Grid2dImgPatches): exact k-NN and radius search in the four metrics against scipy's cKDTree, the
symmetrisations against the reference's formulas, and the graphs against
tests/golden/nngraph.npz (the unmodified PyGSP 0.6.1)."""
import numpy as np
import pytest
from scipy import sparse, spatial

from conftest import csr_from
from oracle import nngraph_oracle as nno

pytestmark = pytest.mark.gpu

METRICS = {"euclidean": 2.0, "manhattan": 1.0, "max_dist": np.inf, "minkowski": 3.0}
SYMS = ("average", "maximum", "fill", "tril", "triu")
SHAPES = {"3x3": (3, 3), "4x2": (4, 2), "5": (5,)}


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch


def _extra(metric):
    return {"order": 3} if metric == "minkowski" else {}


def _device_csr_equal(got, want, rtol=1e-12, exact=False):
    np.testing.assert_array_equal(got.indptr.cpu().numpy(), want.indptr)
    np.testing.assert_array_equal(got.indices.cpu().numpy(), want.indices)
    if exact:
        np.testing.assert_array_equal(got.data.cpu().numpy(), want.data)
    else:
        np.testing.assert_allclose(got.data.cpu().numpy(), want.data, rtol=rtol, atol=0)


# ---------------------------------------------------------------------------- k-NN search
@pytest.mark.parametrize("metric", list(METRICS))
@pytest.mark.parametrize("d", [1, 4, 9, 27, 64, 200])
def test_knn_matches_ckdtree(torch, d, metric):
    from pygsp_b200.graphs import knn_device
    p = METRICS[metric]
    rng = np.random.default_rng(100 + d)
    for k in (1, 10, 32):
        for n in (k + 1, 63, 64, 65, 1000, 20000):
            if n == 20000 and d > 27:
                continue
            X = rng.normal(size=(n, d))
            nn, dist = knn_device(X, k, p=p)
            nn, dist = nn.cpu().numpy(), dist.cpu().numpy()
            rows = np.arange(n) if n <= 1000 else rng.choice(n, 300, replace=False)
            D, NN = spatial.cKDTree(X).query(X[rows], k=k + 1, p=p)
            D, NN = D.reshape(len(rows), -1), NN.reshape(len(rows), -1)
            np.testing.assert_array_equal(nn[rows], NN[:, 1:], err_msg="n=%d k=%d" % (n, k))
            np.testing.assert_allclose(dist[rows], D[:, 1:], rtol=1e-12, atol=0)


@pytest.mark.parametrize("metric", list(METRICS))
def test_knn_ties_and_duplicates(torch, metric):
    from pygsp_b200.graphs import knn_device
    p = METRICS[metric]
    grid = np.stack(np.meshgrid(*[np.arange(3.0)] * 4, indexing="ij"), -1).reshape(-1, 4)
    X = np.concatenate([grid, grid[[0, 5, 17, 40, 80]], grid[[40]]])
    n, k = X.shape[0], 12
    nn1, d1 = knn_device(X, k, p=p)
    nn2, d2 = knn_device(X, k, p=p)
    assert torch.equal(nn1, nn2) and torch.equal(d1, d2)
    nn, dist = nn1.cpu().numpy(), d1.cpu().numpy()
    D, _ = spatial.cKDTree(X).query(X, k=k + 1, p=p)
    if metric == "minkowski":
        np.testing.assert_allclose(dist, D[:, 1:], rtol=1e-12)
    else:
        np.testing.assert_array_equal(dist, D[:, 1:])
    assert not (nn == np.arange(n)[:, None]).any()
    for i in range(n):
        order = np.lexsort((nn[i], dist[i]))
        np.testing.assert_array_equal(order, np.arange(k))
        assert len(set(nn[i])) == k


# --------------------------------------------------------------------------- radius search
def _radius_cloud(rng, n, d, p, per_point=6):
    """A cloud, an isolated far point and a radius with no pair near the boundary."""
    X = rng.normal(size=(n, d))
    X[-1] = 100.0
    D = np.sort(spatial.distance.pdist(X, "minkowski", p=p))
    m = per_point * n // 2
    while D[m + 1] - D[m] <= 4e-12 * D[m]:
        m += 1
    return X, 0.5 * (D[m] + D[m + 1])


@pytest.mark.parametrize("metric", list(METRICS))
@pytest.mark.parametrize("d", [1, 5, 33])
def test_radius_matches_query_ball_point(torch, d, metric):
    from pygsp_b200.graphs import radius_device
    p = METRICS[metric]
    rng = np.random.default_rng(7 + d)
    X, eps = _radius_cloud(rng, 700, d, p)
    R = radius_device(X, eps, p=p)
    R2 = radius_device(X, eps, p=p)
    assert torch.equal(R.indices, R2.indices) and torch.equal(R.data, R2.data)
    indptr, indices, dist = (R.indptr.cpu().numpy(), R.indices.cpu().numpy(),
                             R.data.cpu().numpy())
    lists = spatial.cKDTree(X).query_ball_point(X, r=eps, p=p)
    for i in range(X.shape[0]):
        want = sorted(j for j in lists[i] if j != i)
        got = indices[indptr[i]:indptr[i + 1]]
        np.testing.assert_array_equal(got, want)
        ref = [nno.minkowski(X[i], X[j], p) for j in want]
        np.testing.assert_allclose(dist[indptr[i]:indptr[i + 1]], ref, rtol=1e-12)
    assert indptr[-1] - indptr[-2] == 0          # the far point has no neighbour


def test_radius_without_neighbours_raises(torch):
    from pygsp_b200.graphs import NNGraph
    X = np.arange(40.0).reshape(20, 2) * 10
    with pytest.raises(ValueError, match="No neighbors found"):
        NNGraph(X, NNtype="radius", epsilon=1e-3, rescale=False, center=False)


# ------------------------------------------------------------------------ symmetrisation
@pytest.mark.parametrize("method", SYMS)
def test_symmetrize_device_matches_reference(torch, method):
    from pygsp_b200.graphs import DeviceCSR, symmetrize_device
    rng = np.random.default_rng(3)
    n = 400
    W = sparse.random(n, n, density=0.02, random_state=5, format="csr",
                      data_rvs=lambda s: rng.uniform(0.1, 2.0, s))
    W = W.tolil()
    W[:50, :50] = W.T.tocsr()[:50, :50]                    # a block of exact mirrors: ties
    W = W.tocsr()
    W.sort_indices()
    W.data[1::11] = W.data[1::11].round(1)
    W.data[::7] = 0.0                                      # stored zeros
    assert (W.data == 0).any()
    want = sparse.csr_matrix(nno.symmetrize(W, method))
    want.eliminate_zeros()
    want.sort_indices()
    dev = torch.device("cuda")
    got = symmetrize_device(DeviceCSR.from_scipy(W, torch.float64, dev), method)
    _device_csr_equal(got, want, exact=True)


# ------------------------------------------------------------------ graphs vs the reference
@pytest.mark.parametrize("nntype", ["knn", "radius"])
@pytest.mark.parametrize("metric", list(METRICS))
@pytest.mark.parametrize("d", [1, 3, 8, 27])
def test_nngraph_matches_golden(torch, golden, nntype, metric, d):
    from pygsp_b200.graphs import NNGraph
    z = golden("nngraph")
    X = z["X_d%d" % d]
    eps = float(z["eps_d%d_%s" % (d, metric)])
    for sym in SYMS:
        tag = "nn_%s_d%d_%s_%s" % (nntype, d, metric, sym)
        G = NNGraph(X, NNtype=nntype, dist_type=metric, epsilon=eps, symmetrize_type=sym,
                    dtype=np.float64, **_extra(metric))
        want = csr_from(z, tag + "_W")
        _device_csr_equal(G.W, want)
        np.testing.assert_allclose(G.sigma, z[tag + "_sigma"], rtol=1e-13)
        assert (G.NNtype, G.dist_type, G.symmetrize_type, G.epsilon) == (nntype, metric, sym, eps)


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("img", ["gray", "rgb"])
def test_patch_graphs_match_golden(torch, golden, img, shape):
    from pygsp_b200.graphs import Grid2dImgPatches, ImgPatches
    z = golden("nngraph")
    im = z["img_" + img]
    tag = "%s_%s" % (img, shape)
    G = ImgPatches(im, patch_shape=SHAPES[shape], dtype=np.float64)
    np.testing.assert_array_equal(G.Xin.cpu().numpy(), z["ip_%s_X" % tag])
    _device_csr_equal(G.W, csr_from(z, "ip_%s_W" % tag))
    np.testing.assert_allclose(G.sigma, z["ip_%s_sigma" % tag], rtol=1e-13)
    G2 = Grid2dImgPatches(im, patch_shape=SHAPES[shape], dtype=np.float64)
    _device_csr_equal(G2.W, csr_from(z, "g2ip_%s_W" % tag))
    G3 = Grid2dImgPatches(im, aggregate=lambda Wp, Wg: Wp.maximum(Wg), patch_shape=SHAPES[shape],
                          dtype=np.float64)
    want = csr_from(z, "ip_%s_W" % tag).maximum(nno.grid2d(im.shape[0], im.shape[1]))
    np.testing.assert_allclose(G3.W.toarray(), want.toarray(), rtol=1e-12, atol=0)


def test_reference_nngraph_calls(torch):
    """The calls of the reference's tests/test_graphs.py::test_nngraph, verbatim."""
    from pygsp_b200 import graphs
    n_vertices = 30
    rng = np.random.default_rng(42)
    Xin = rng.normal(size=(n_vertices, 3))
    dist_types = ["euclidean", "manhattan", "max_dist", "minkowski"]
    for dist_type in dist_types:
        if dist_type != "minkowski":
            graphs.NNGraph(Xin, NNtype="radius", dist_type=dist_type, epsilon=0.1)
            graphs.NNGraph(Xin, NNtype="knn", dist_type=dist_type)
        if dist_type != "max_dist":
            graphs.NNGraph(Xin, use_flann=True, NNtype="knn", dist_type=dist_type)


def test_argument_errors(torch):
    from pygsp_b200.graphs import NNGraph
    X = np.random.default_rng(0).normal(size=(20, 4))
    with pytest.raises(ValueError):
        NNGraph(X, k=20, NNtype="radius")
    with pytest.raises(ValueError):
        NNGraph(X, NNtype="kmeans")
    with pytest.raises(ValueError):
        NNGraph(X, dist_type="cosine")
    with pytest.raises(ValueError):
        NNGraph(X, dist_type="minkowski", order=0.5)
    with pytest.raises(ValueError):
        NNGraph(X, symmetrize_type="sum")


# ------------------------------------------------------------------------------- scale
def test_scale_200k_points(torch):
    from pygsp_b200.graphs import NNGraph, knn_device
    rng = np.random.default_rng(11)
    n, d, k = 200_000, 32, 10
    X = rng.normal(size=(n, d))
    nn, _ = knn_device(X, k)
    nn = nn.cpu().numpy()
    for i in rng.choice(n, 500, replace=False):
        d2 = np.sum((X - X[i]) ** 2, axis=1)
        d2[i] = np.inf
        want = np.lexsort((np.arange(n), d2))[:k]
        np.testing.assert_array_equal(nn[i], want)
    G64 = NNGraph(X, k=k, dtype=np.float64)
    G32 = NNGraph(X, k=k, dtype=np.float32)
    assert torch.equal(G64.W.indptr, G32.W.indptr) and torch.equal(G64.W.indices, G32.W.indices)
    np.testing.assert_allclose(G32.W.data.cpu().numpy(), G64.W.data.cpu().numpy(), rtol=2e-7)


# ----------------------------------------------------------------------------- routing
def test_backend_routing(torch, monkeypatch):
    from pygsp_b200 import _native as nat
    from pygsp_b200.graphs import NNGraph
    seen = []
    real = nat.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)
    monkeypatch.setattr(nat, "call", spy)
    rng = np.random.default_rng(1)
    NNGraph(rng.uniform(size=(500, 2)), k=6)
    assert "gsp_knn_grid" in seen and "gsp_knn_brute" not in seen
    seen.clear()
    NNGraph(rng.normal(size=(500, 8)), k=6)
    assert "gsp_knn_brute" in seen and "gsp_knn_grid" not in seen
    seen.clear()
    NNGraph(rng.uniform(size=(500, 3)), k=6, dist_type="manhattan")
    assert "gsp_knn_brute" in seen
    seen.clear()
    NNGraph(rng.normal(size=(300, 5)), k=40)                 # k > 32: host cKDTree
    assert "gsp_knn_brute" not in seen and "gsp_knn_grid" not in seen
