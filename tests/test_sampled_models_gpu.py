"""Sampled graph models on the device (pygsp_b200/graphs/sampled.py): the segmented neighbour
search against the unsegmented one, the exact-size subset sampler against its serial oracle,
and Community, SwissRoll, Sphere, Cube and TwoMoons against the PyGSP 0.6.1 fixture
tests/golden/sampled_models.npz."""
import hashlib
import json

import numpy as np
import pytest
from scipy import sparse, spatial, stats

from conftest import csr_from

pytestmark = pytest.mark.gpu

GOLD = "sampled_models"


def _sym(g, prefix):
    """The fixture's adjacency: it stores the strict upper triangle T of a symmetric W."""
    T = csr_from(g, prefix)
    return (T + T.T).tocsr()


def _same(a, g, key):
    """a's float64 C-order bytes have the fixture's SHA-256."""
    got = hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()
    assert got == str(g[key]), key


@pytest.fixture(scope="module")
def gsp():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


def _build(gsp, golden, name, **extra):
    g = golden(GOLD)
    args = json.loads(str(g[name + "_args"]))
    return getattr(gsp.graphs, args["model"])(**args["kwargs"], **extra)


# ------------------------------------------------------------------ segmented search -------
SIZES = [0, 1, 63, 64, 65, 0, 700] + [3] * 30 + [2, 1, 130]


def _cloud(sizes, d, seed):
    rng = np.random.default_rng(seed)
    n = int(np.sum(sizes))
    # a coarse lattice: many tied distances, so the (distance, id) order is exercised
    return np.round(rng.uniform(0, 4, (n, d)) * 2) / 2


@pytest.mark.parametrize("p", [1.0, 2.0, np.inf, 3.0])
@pytest.mark.parametrize("d", [2, 5])
def test_segmented_knn_equals_per_segment_search(gsp, p, d):
    graphs = gsp.graphs
    X = _cloud(SIZES, d, 1)
    k = 4
    nn, dist = graphs.knn_segments_device(X, SIZES, k, p)
    nn, dist = nn.cpu().numpy(), dist.cpu().numpy()
    start = 0
    for s in SIZES:
        seg = slice(start, start + s)
        if s >= 2:
            kk = min(k, s - 1)
            ref_nn, ref_d = _brute(gsp, X[seg], kk, p)
            np.testing.assert_array_equal(nn[seg, :kk], ref_nn.cpu().numpy() + start)
            np.testing.assert_array_equal(dist[seg, :kk], ref_d.cpu().numpy())
            assert (nn[seg, kk:] == -1).all() and (dist[seg, kk:] == 0).all()
        elif s == 1:
            assert (nn[seg] == -1).all()
        start += s


def _brute(gsp, X, k, p):
    """gsp_knn_brute itself (knn_device takes the cell grid for Euclidean 2-D / 3-D)."""
    import torch
    nat = gsp._native
    pts = torch.as_tensor(X, dtype=torch.float64, device="cuda").contiguous()
    nn = torch.empty((X.shape[0], k), dtype=torch.int32, device="cuda")
    dist = torch.empty((X.shape[0], k), dtype=torch.float64, device="cuda")
    nat.call("gsp_knn_brute", nat.i64(X.shape[0]), nat.i32(X.shape[1]), pts, nat.i32(k),
             nat.f64(p), nn, dist, nat.stream_ptr())
    return nn, dist


@pytest.mark.parametrize("p", [1.0, 2.0, np.inf, 3.0])
@pytest.mark.parametrize("d", [2, 17])
def test_segmented_radius_equals_per_segment_search(gsp, p, d):
    graphs = gsp.graphs
    from scipy.spatial.distance import pdist
    X = _cloud(SIZES, d, 2)
    big = X[193:893]                   # the 700-point segment: eps at its 2 % distance quantile
    eps = float(np.quantile(pdist(big, "minkowski", p=p) if np.isfinite(p)
                            else pdist(big, "chebyshev"), 0.02))
    D = graphs.radius_segments_device(X, SIZES, eps, p).to_scipy()
    start, total = 0, 0
    for s in SIZES:
        if s:
            ref = graphs.radius_device(X[start:start + s], eps, p).to_scipy()
            blk = D[start:start + s]
            assert blk[:, :start].nnz == 0 and blk[:, start + s:].nnz == 0
            blk = blk[:, start:start + s].tocsr()
            np.testing.assert_array_equal(blk.indptr, ref.indptr)
            np.testing.assert_array_equal(blk.indices, ref.indices)
            np.testing.assert_array_equal(blk.data, ref.data)
            total += ref.nnz
        start += s
    assert D.nnz == total > 0


def test_segment_spanning_many_ctas(gsp):
    graphs = gsp.graphs
    sizes = [5, 3000, 7]
    X = _cloud(sizes, 3, 3)
    nn, dist = graphs.knn_segments_device(X, sizes, 6, 2)
    ref_nn, ref_d = _brute(gsp, X[5:3005], 6, 2.0)
    np.testing.assert_array_equal(nn[5:3005].cpu().numpy(), ref_nn.cpu().numpy() + 5)
    np.testing.assert_array_equal(dist[5:3005].cpu().numpy(), ref_d.cpu().numpy())


# ------------------------------------------------------------------ exact-size subsets -----
def _spaces():
    from pygsp_b200.graphs.random_graphs import RECT, TRI_STRICT
    return [([(TRI_STRICT, 45, 10, 0, 0)], 17), ([(TRI_STRICT, 190, 20, 10, 10)], 0),
            ([(RECT, 200, 10, 10, 0)], 200), ([(TRI_STRICT, 4950, 100, 30, 30)], 4000),
            ([(RECT, 2000, 20, 130, 10), (RECT, 30000, 100, 150, 30)], 300)]


@pytest.mark.parametrize("max_blocks", [0, 3])
def test_subset_sampler_matches_oracle(gsp, monkeypatch, max_blocks):
    from oracle import sampled_models_oracle as smo
    from pygsp_b200.graphs import sampled
    monkeypatch.setattr(sampled, "_MAX_BLOCKS", max_blocks)
    for key in (5, 2 ** 62 + 11):
        rows, cols, attempt = sampled.subset_device(450, _spaces(), key)
        ref_r, ref_c, ref_attempt = smo.subset_pairs(450, _spaces(), key)
        assert attempt == ref_attempt
        np.testing.assert_array_equal(rows.cpu().numpy(), ref_r)
        np.testing.assert_array_equal(cols.cpu().numpy(), ref_c)


def test_subset_sampler_exact_counts_in_a_large_space(gsp):
    """One space of 4.5e9 pairs (a 30000 x 150000 rectangle): exactly n distinct pairs."""
    from pygsp_b200.graphs import sampled
    from pygsp_b200.graphs.random_graphs import RECT
    n = 123457
    rows, cols, _ = sampled.subset_device(180000, [([(RECT, 30000 * 150000, 150000, 150000, 0)],
                                                    n)], 99)
    r, c = rows.cpu().numpy()[0::2].astype(np.int64), cols.cpu().numpy()[0::2].astype(np.int64)
    assert r.size == n and (r >= 150000).all() and (c < 150000).all()
    assert np.unique(r * 180000 + c).size == n


# ------------------------------------------------------------------ Community --------------
def _max_ulps_of_eps2(coords, pairs, eps):
    d2 = np.array([np.sum((coords[i] - coords[j]) ** 2) for i, j in pairs])
    return np.abs(d2 - eps * eps) / np.spacing(eps * eps)


@pytest.mark.parametrize("name", ["community_exact", "community_exact_small"])
def test_community_exact_case_equals_reference(gsp, golden, name):
    g = golden(GOLD)
    G = _build(gsp, golden, name, dtype=np.float64)
    _same(G.coords, g, name + "_coords_sha256")
    ref = _sym(g, name + "_W")
    W = G.W.to_scipy()
    diff = (abs(W - ref) > 0).tocoo()
    pairs = list(zip(diff.row.tolist(), diff.col.tolist()))
    eps = float(json.loads(str(g[name + "_info_json"]))["epsilon"])
    if pairs:
        assert _max_ulps_of_eps2(G.coords, pairs, eps).max() <= 4
    assert len(pairs) <= 4
    assert W.nnz > 1000 and (W.data == 1).all()
    for key in ("node_com", "comm_sizes", "com_coords"):
        np.testing.assert_array_equal(G.info[key], g["%s_info_%s" % (name, key)])


def _structure(W, N):
    W = W.to_scipy()
    assert (W.data == 1).all()
    assert (W != W.T).nnz == 0
    assert W.diagonal().sum() == 0
    return W


def _block_counts(G):
    com = np.asarray(G.info["node_com"])
    coo = sparse.tril(G.W.to_scipy(), k=-1).tocoo()
    a, b = com[coo.row], com[coo.col]
    out = np.zeros((G.Nc, G.Nc), dtype=np.int64)
    np.add.at(out, (np.maximum(a, b), np.minimum(a, b)), 1)
    return out


@pytest.mark.parametrize("case", ["default", "dense_world", "comm_density"])
def test_community_sampled_cases(gsp, golden, case):
    """Exact totals, symmetric unit W without loops, and inter-community block counts summed
    over the fixture's seeds consistent with the reference's (chi-square homogeneity)."""
    g = golden(GOLD)
    kwargs = json.loads(str(g["blocks_%s_args" % case]))
    ours = []
    for seed in g["blocks_%s_seeds" % case]:
        G = gsp.graphs.Community(seed=int(seed), **kwargs)
        W = _structure(G.W, G.N)
        sizes = G.info["comm_sizes"]
        blocks = _block_counts(G)
        M = (G.N ** 2 - np.sum(sizes ** 2)) / 2
        inter = blocks.sum() - np.trace(blocks)
        assert inter == int(G.info["world_density"] * M)
        if "comm_density" in kwargs:
            np.testing.assert_array_equal(
                np.diag(blocks), [int(kwargs["comm_density"] * (s * (s - 1) / 2)) for s in sizes])
        assert W.nnz == 2 * blocks.sum()
        ours.append(blocks)
    ours, ref = np.sum(ours, axis=0), g["blocks_" + case].sum(axis=0)
    lower = np.tril_indices(ref.shape[0], -1)
    assert ours[lower].sum() == ref[lower].sum()
    table = np.stack([ours[lower], ref[lower]])
    table = table[:, table.sum(axis=0) > 0]
    if table.shape[1] > 1:
        assert stats.chi2_contingency(table).pvalue > 1e-6


def test_community_is_a_function_of_the_seed(gsp):
    a = gsp.graphs.Community(N=500, world_density=0.1, seed=3).W.to_scipy()
    b = gsp.graphs.Community(N=500, world_density=0.1, seed=3).W.to_scipy()
    assert (a != b).nnz == 0


def test_community_layout_equals_reference(gsp, golden):
    g = golden(GOLD)
    for name in ("community_sizes", "community_exact_small"):
        G = _build(gsp, golden, name)
        G.set_coordinates("community2D", seed=7)
        _same(G.coords, g, name + "_layout_sha256")


def test_community_knn_builds_the_documented_graph(gsp, golden):
    """The reference's k_neigh branch adds no intra edge (fixture: 0 entries); this one builds
    the union of each vertex's k nearest neighbours in its community."""
    g = golden(GOLD)
    assert g["community_knn_empty_W_indices"].size == 0
    G = _build(gsp, golden, "community_knn_empty", dtype=np.float64)
    W = _structure(G.W, G.N)
    sizes, start, ref = G.info["comm_sizes"], 0, sparse.lil_matrix((G.N, G.N))
    for s in sizes:
        _, nn = spatial.cKDTree(G.coords[start:start + s]).query(G.coords[start:start + s], k=6)
        for i in range(s):
            for j in nn[i, 1:]:
                ref[start + i, start + j] = ref[start + j, start + i] = 1
        start += s
    ref = ref.tocsr()
    assert abs(W - ref).nnz <= 4      # only exact distance ties may choose differently
    assert W.nnz >= 5 * G.N


def test_community_refuses_2_31_entries_before_the_fill(gsp, monkeypatch):
    """Community(N=10^7) with the defaults has more than 2^31 intra entries: ValueError after
    the segmented count, before the fill."""
    nat = gsp._native
    called = []
    real = nat.call

    def spy(name, *args):
        called.append(name)
        return real(name, *args)
    monkeypatch.setattr(nat, "call", spy)
    with pytest.raises(ValueError, match="2\\^31"):
        gsp.graphs.Community(N=10 ** 7, seed=0)
    assert "gsp_radius_count_seg" in called
    assert "gsp_radius_fill_seg_f64" not in called and "gsp_subset_select" not in called


# ------------------------------------------------------------------ SwissRoll --------------
SWISS = ["swissroll_400_3d", "swissroll_1000_3d", "swissroll_400_2d", "swissroll_1000_2d",
         "swissroll_noise", "swissroll_classic"]


@pytest.mark.parametrize("name", SWISS)
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_swissroll_equals_reference(gsp, golden, name, dtype):
    g = golden(GOLD)
    G = _build(gsp, golden, name, dtype=dtype)
    from oracle import sampled_models_oracle as smo
    _same(G.coords, g, name + "_coords_sha256")
    _same(G.x, g, name + "_x_sha256")
    # the reference's weights: the fixture keeps their structure and digest, which the
    # restatement reproduces (tests/test_sampled_models_cpu.py)
    T = smo.swissroll_reference(G.coords, G.s, G.thresh)
    np.testing.assert_array_equal(T.indptr, g[name + "_W_indptr"])
    np.testing.assert_array_equal(T.indices, g[name + "_W_indices"])
    ref, W = (T + T.T).tocsr(), G.W.to_scipy().astype(np.float64)
    thresh = G.thresh
    # the reference's Gram-expansion distances: |d^2 error| <= 8 u max|x|^2, so a weight w
    # near the threshold moves by at most w * that / (2 s^2) relatively
    tol = 8 * np.finfo(np.float64).eps * 2 * np.max(np.abs(G.coords)) ** 2 / (2 * G.s ** 2)
    only = ((W != 0).astype(int) - (ref != 0).astype(int)).tocoo()
    for i, j in zip(only.row, only.col):
        w = max(W[i, j], ref[i, j])
        assert abs(w - thresh) <= 2 * tol * thresh + (1e-6 if dtype == np.float32 else 0), (i, j)
    both = W.multiply(ref != 0).tocsr()
    refb = ref.multiply(W != 0).tocsr()
    both.sort_indices()
    refb.sort_indices()
    np.testing.assert_allclose(both.data, refb.data, rtol=1e-12 if dtype == np.float64 else 2e-6)
    assert W.nnz > 0


def test_swissroll_matches_direct_difference_oracle(gsp):
    from oracle import sampled_models_oracle as smo
    G = gsp.graphs.SwissRoll(N=5000, seed=11, dtype=np.float64)
    ref = smo.swissroll_weights(G.coords, G.s, G.thresh)
    W = G.W.to_scipy()
    W.sort_indices()
    ref.sort_indices()
    np.testing.assert_array_equal(W.indices, ref.indices)
    np.testing.assert_allclose(W.data, ref.data, rtol=1e-14)


def test_swissroll_without_threshold_keeps_every_positive_weight(gsp):
    G = gsp.graphs.SwissRoll(N=300, thresh=0, s=0.3, seed=2, dtype=np.float64)
    from oracle import sampled_models_oracle as smo
    ref = smo.swissroll_weights(G.coords, G.s, 0.0)
    W = G.W.to_scipy()
    assert W.nnz == ref.nnz
    # exp(-x) up to x = 745 scales the rounding of d^2 by x, and subnormal weights keep no
    # relative precision
    np.testing.assert_allclose(W.toarray(), ref.toarray(), rtol=1e-12, atol=1e-300)


# ------------------------------------------------------------------ NN models --------------
@pytest.mark.parametrize("name", ["sphere_s0", "sphere_s1", "sphere_4d", "cube_3d_s0",
                                  "cube_3d_s1", "cube_2d", "twomoons_s0", "twomoons_s1"])
def test_nn_models_equal_reference(gsp, golden, name):
    g = golden(GOLD)
    G = _build(gsp, golden, name, dtype=np.float64)
    _same(G.coords, g, name + "_coords_sha256")
    ref, W = _sym(g, name + "_W"), G.W.to_scipy()
    assert (abs(W - ref) > 1e-12).nnz == 0
    assert W.nnz == ref.nnz
    if name.startswith("twomoons"):
        np.testing.assert_array_equal(G.labels, g[name + "_labels"])
