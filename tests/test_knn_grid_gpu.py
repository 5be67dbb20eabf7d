"""The cell-grid k-NN search (gsp_knn_grid, behind graphs.knn_device for Euclidean 2-D / 3-D
clouds) against the exhaustive search gsp_knn_brute(p = 2), which sums the same squares by FMA in
the same order: ids and distances must be the same bits, on the clouds of tests/knn_clouds.py
(tied lattices, duplicates, degenerate boxes, clusters) and at sizes around k + 1 and multiples
of 256.  Where every squared distance is exact in float64, a NumPy brute force gives the true
(distance, id) order as well.  At graph level, NNGraph's W from the grid path equals the W built
from the exhaustive lists."""
import numpy as np
import pytest

import knn_clouds

pytestmark = pytest.mark.gpu

KS = (1, 10, 32)
# k = 21, 25, 26 put the k-th distance of many rows of the permuted 31 x 31 lattice on a cell
# face, with a lower-id tie beyond it
CASES = [(name, k) for name in knn_clouds.NAMES for k in KS
         if knn_clouds.cloud(name)[0].shape[0] > k]
CASES += [(name, k) for name in ("lattice2d_perm", "lattice2d_perm_shift") for k in (21, 25, 26)]


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch


@pytest.fixture
def grid_calls(monkeypatch):
    """Names of the native calls made, to show that the grid search is the one tested."""
    from pygsp_b200 import _native as nat
    seen = []
    real = nat.call

    def spy(name, *args):
        seen.append(name)
        return real(name, *args)
    monkeypatch.setattr(nat, "call", spy)
    return seen


def _exhaustive(torch, X, k):
    from pygsp_b200 import _native as nat
    pts = torch.as_tensor(np.ascontiguousarray(X), device="cuda")
    n, dim = pts.shape
    nn = torch.empty((n, k), dtype=torch.int32, device="cuda")
    dist = torch.empty((n, k), dtype=torch.float64, device="cuda")
    nat.call("gsp_knn_brute", nat.i64(n), nat.i32(dim), pts, nat.i32(k), nat.f64(2.0), nn, dist,
             nat.stream_ptr(pts.device))
    return nn, dist


def _numpy_lists(X, k, rows):
    """(ids, distances) of `rows` by float64 squares, ordered by (distance, id)."""
    n = X.shape[0]
    ids = np.empty((len(rows), k), dtype=np.int64)
    dist = np.empty((len(rows), k))
    for r, i in enumerate(rows):
        d2 = ((X - X[i]) ** 2).sum(axis=1)
        d2[i] = np.inf
        ids[r] = np.lexsort((np.arange(n), d2))[:k]
        dist[r] = np.sqrt(d2[ids[r]])
    return ids, dist


def _check(torch, X, k, ppc, seen):
    from pygsp_b200.graphs import knn_device
    nn, dist = knn_device(X, k, points_per_cell=ppc)
    assert "gsp_knn_grid" in seen and "gsp_knn_brute" not in seen
    nn2, dist2 = knn_device(X, k, points_per_cell=ppc)
    assert torch.equal(nn, nn2) and torch.equal(dist, dist2), "two runs differ"
    bn, bd = _exhaustive(torch, X, k)
    bad = (nn != bn).any(dim=1).nonzero().flatten()[:5].tolist()
    assert torch.equal(nn, bn), "rows %s differ from the exhaustive search" % bad
    assert torch.equal(dist, bd)
    if knn_clouds.exact(X):
        n = X.shape[0]
        rows = np.arange(n) if n <= 3000 else np.unique(np.concatenate(
            [np.random.default_rng(n).choice(n, 400, replace=False), [0, n - 1]]))
        ids, d = _numpy_lists(np.asarray(X), k, rows)
        np.testing.assert_array_equal(nn.cpu().numpy()[rows], ids)
        np.testing.assert_array_equal(dist.cpu().numpy()[rows], d)


@pytest.mark.parametrize("name,k", CASES)
def test_grid_equals_exhaustive_search(torch, grid_calls, name, k):
    X, ppc = knn_clouds.cloud(name)
    _check(torch, X, k, ppc, grid_calls)


@pytest.mark.parametrize("dim", [2, 3])
@pytest.mark.parametrize("k", KS)
def test_grid_at_block_edge_sizes(torch, grid_calls, dim, k):
    """n = k + 1 (every other point is a neighbour) and n next to multiples of the 256-thread
    blocks, on small-integer clouds full of ties and duplicates."""
    for n in sorted({k + 1, 255, 256, 257, 511, 512, 513, 769}):
        X = np.random.default_rng(n * dim + k).integers(-3, 4, (n, dim)).astype(np.float64)
        grid_calls.clear()
        _check(torch, X, k, 3.0, grid_calls)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("name", ["lattice2d_perm", "lattice3d_perm_shift", "repeat5",
                                  "two_clusters", "line_z_3d", "spread1e-14_2d",
                                  "cluster_outliers", "box_max"])
def test_nngraph_w_equals_w_of_exhaustive_lists(torch, name, dtype):
    """NNGraph's k-NN adjacency (grid path) is, bit for bit, gsp_knn_to_csr_* + 'average' of the
    exhaustive lists with sigma their mean distance.  (Not on clouds where all k = 10 distances
    are 0: sigma = 0 makes every weight NaN, which Graph refuses.)"""
    from pygsp_b200 import _native as nat
    from pygsp_b200.graphs import DeviceCSR, NNGraph, symmetrize_device
    X, _ = knn_clouds.cloud(name)
    k = 10
    G = NNGraph(X, k=k, center=False, rescale=False, dtype=dtype)
    nn, dist = _exhaustive(torch, X, k)
    sigma = float(dist.mean().item())
    assert G.sigma == sigma
    n = X.shape[0]
    dt = torch.float32 if dtype == np.float32 else torch.float64
    indptr = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    indices = torch.empty(n * k, dtype=torch.int32, device="cuda")
    data = torch.empty(n * k, dtype=dt, device="cuda")
    nat.call("gsp_knn_to_csr_" + nat.suffix(dt), nat.i64(n), nat.i32(k), nn, dist, nat.f64(sigma),
             indptr, indices, data, nat.stream_ptr(nn.device))
    W = symmetrize_device(DeviceCSR(indptr, indices, data, (n, n)), "average")
    assert torch.equal(G.W.indptr, W.indptr) and torch.equal(G.W.indices, W.indices)
    assert G.W.data.dtype == dt and torch.equal(G.W.data, W.data)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_non_finite_points_are_refused(torch, bad):
    from pygsp_b200.graphs import NNGraph, knn_device, radius_device
    for dim in (5, 3, 2):        # the exhaustive search, then the grid
        X = np.random.default_rng(dim).uniform(size=(100, dim))
        X[17, dim - 1] = bad
        with pytest.raises(ValueError, match="finite"):
            knn_device(X, 5)
        with pytest.raises(ValueError, match="finite"):
            knn_device(torch.as_tensor(X, device="cuda"), 5)
        with pytest.raises(ValueError, match="finite"):
            radius_device(X, 0.1)
        with pytest.raises(ValueError, match="finite"):
            NNGraph(X, k=5, center=False, rescale=False)
