"""Tree multiresolution on the device (csrc/tree.cu, reduction.tree_multiresolution): every level
bit for bit against the NumPy rules of oracle/tree_oracle.py (kept vertices, W's structure and
values, root, coordinates, mr) for each reduction method in float64 and float32, on paths up to
10^6 vertices (depth 10^6 - 1), directed paths, stars, a comet, low stretch trees and relabelled
random trees with weights over six decades; the rooting against BFS; the errors; determinism; a
pyramid analysis / synthesis round trip; and the spectra of compute_full_eigen."""
import numpy as np
import pytest
from scipy import sparse

from oracle import pygsp_oracle as orc
from oracle import tree_oracle as tro

pytestmark = pytest.mark.gpu

DTYPES = (np.float64, np.float32)


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


def _random(gsp, n, seed, dtype):
    W = tro.random_tree(n, seed)
    coords = np.random.default_rng(seed + 1).random((n, 2))
    return gsp.graphs.Graph(W, coords=coords, dtype=dtype)


# (name, builder(gsp, dtype), Nlevel, root): small graphs run past their depth (one-vertex levels)
GRAPHS = [
    ("path1", lambda g, dt: g.graphs.Path(1, dtype=dt), 3, 0),
    ("path2", lambda g, dt: g.graphs.Path(2, dtype=dt), 3, None),
    ("path3", lambda g, dt: g.graphs.Path(3, dtype=dt), 3, None),
    ("path17", lambda g, dt: g.graphs.Path(17, dtype=dt), 8, None),
    ("path17_root0", lambda g, dt: g.graphs.Path(17, dtype=dt), 8, 0),
    ("path1e6", lambda g, dt: g.graphs.Path(10 ** 6, dtype=dt), 4, None),
    ("path16_directed", lambda g, dt: g.graphs.Path(16, directed=True, dtype=dt), 6, None),
    ("star10", lambda g, dt: g.graphs.Star(10, dtype=dt), 3, None),
    ("star1e5", lambda g, dt: g.graphs.Star(10 ** 5, dtype=dt), 3, None),
    ("comet", lambda g, dt: g.graphs.Comet(32, 12, dtype=dt), 6, None),
    ("lst1", lambda g, dt: g.graphs.LowStretchTree(1, dtype=dt), 3, None),
    ("lst2", lambda g, dt: g.graphs.LowStretchTree(2, dtype=dt), 4, None),
    ("lst3", lambda g, dt: g.graphs.LowStretchTree(3, dtype=dt), 6, None),
    ("lst6", lambda g, dt: g.graphs.LowStretchTree(6, dtype=dt), 8, None),
    ("lst10", lambda g, dt: g.graphs.LowStretchTree(10, dtype=dt), 3, None),
    ("random1e3", lambda g, dt: _random(g, 1000, 7, dt), 12, 5),
    ("random2e6", lambda g, dt: _random(g, 2 * 10 ** 6, 11, dt), 3, None),
]
_BUILT = {}


def _graph(gsp, name, dtype):
    key = (name, np.dtype(dtype).name)
    if key not in _BUILT:
        _BUILT.clear()                       # keep one large graph alive at a time
        builder = dict((g[0], g[1]) for g in GRAPHS)[name]
        _BUILT[key] = builder(gsp, dtype)
    return _BUILT[key]


def _default_root(G, root):
    return root if root is not None else getattr(G, "root", 1)


def _host_support(G):
    return G._symmetric_adjacency().to_scipy()


def _check_levels(G, Gs, sub, levels, nlevel):
    assert Gs[0] is G and len(Gs) == nlevel + 1 and len(sub) == nlevel
    np.testing.assert_array_equal(G.mr["idx"], np.arange(G.N))
    np.testing.assert_array_equal(G.mr["orig_idx"], np.arange(G.N))
    for i, lev in enumerate(levels):
        H, keep = Gs[i + 1], sub[i]
        assert keep.dtype == np.int64
        np.testing.assert_array_equal(keep, lev["keep"])
        S, R = H.W.to_scipy(), lev["W"]
        assert S.shape == R.shape and S.dtype == R.dtype
        np.testing.assert_array_equal(S.indptr, R.indptr)
        np.testing.assert_array_equal(S.indices, R.indices)
        np.testing.assert_array_equal(S.data, R.data)
        assert H.root == lev["root"]
        assert H.dtype == G.dtype and H.lap_type == G.lap_type and H.device == G.device
        if hasattr(G, "coords"):
            np.testing.assert_array_equal(H.coords, np.asarray(G.coords)[lev["orig_idx"]])
        np.testing.assert_array_equal(H.mr["idx"], keep)
        np.testing.assert_array_equal(H.mr["orig_idx"], lev["orig_idx"])
        assert H.mr["level"] == i


@pytest.mark.parametrize("dtype", DTYPES, ids=["f64", "f32"])
@pytest.mark.parametrize("name,nlevel,root", [(g[0], g[2], g[3]) for g in GRAPHS],
                         ids=[g[0] for g in GRAPHS])
def test_levels_match_the_oracle(gsp, name, nlevel, root, dtype):
    G = _graph(gsp, name, dtype)
    r = _default_root(G, root)
    Ws = _host_support(G)
    for method in tro.METHODS:
        Gs, sub = gsp.reduction.tree_multiresolution(G, nlevel, reduction_method=method, root=root)
        levels = tro.tree_multiresolution_levels(Ws, nlevel, method, r, dtype=dtype)
        _check_levels(G, Gs, sub, levels, nlevel)


@pytest.mark.parametrize("name,root", [(g[0], g[3]) for g in GRAPHS], ids=[g[0] for g in GRAPHS])
def test_rooting_matches_bfs(gsp, name, root):
    G = _graph(gsp, name, np.float64)
    r = _default_root(G, root)
    depth, parent = gsp.reduction._tree_depths(G, r)
    d_ref, p_ref, _ = tro.bfs_depths(tro.symmetric_support(_host_support(G)), r)
    np.testing.assert_array_equal(depth.cpu().numpy(), d_ref)
    np.testing.assert_array_equal(parent.cpu().numpy(), p_ref)


def test_path_depth_is_n_minus_one(gsp):
    G = gsp.graphs.Path(10 ** 6, dtype=np.float32)
    depth, parent = gsp.reduction._tree_depths(G, 0)
    np.testing.assert_array_equal(depth.cpu().numpy(), np.arange(10 ** 6))
    np.testing.assert_array_equal(parent.cpu().numpy(), np.maximum(np.arange(10 ** 6) - 1, 0))


def test_one_vertex_levels_repeat(gsp):
    G = gsp.graphs.Star(10, dtype=np.float64)          # root 1 is a leaf: 9 vertices, then 1
    Gs, sub = gsp.reduction.tree_multiresolution(G, 4)
    assert [H.N for H in Gs] == [10, 9, 1, 1, 1]
    for H, keep in zip(Gs[2:], sub[1:]):
        np.testing.assert_array_equal(keep, [0])
        assert H.W.nnz == 0 and H.root == 0
    np.testing.assert_array_equal(Gs[-1].mr["orig_idx"], [1])


def test_errors(gsp):
    red = gsp.reduction
    with pytest.raises(ValueError, match="tree"):
        red.tree_multiresolution(gsp.graphs.Ring(8), 1, root=0)
    P = sparse.diags([np.ones(4), np.ones(4)], [-1, 1], shape=(5, 5))
    two = gsp.graphs.Graph(sparse.block_diag([P, P]).tocsr())
    with pytest.raises(ValueError, match="Graph is not connected"):
        red.tree_multiresolution(two, 1, root=0)
    G = gsp.graphs.Path(8)
    with pytest.raises(ValueError, match="Unknown graph reduction method."):
        red.tree_multiresolution(G, 1, reduction_method="kron")
    for bad in (-1, 8):
        with pytest.raises(ValueError):
            red.tree_multiresolution(G, 1, root=bad)
    with pytest.raises(ValueError):
        red.tree_multiresolution(gsp.graphs.Path(1), 1)   # default root 1 is not a vertex


def test_two_calls_are_bit_identical(gsp):
    G = _random(gsp, 10 ** 5, 3, np.float32)
    a, sa = gsp.reduction.tree_multiresolution(G, 4, root=17)
    b, sb = gsp.reduction.tree_multiresolution(G, 4, root=17)
    for x, y, kx, ky in zip(a[1:], b[1:], sa, sb):
        np.testing.assert_array_equal(kx, ky)
        for f in ("indptr", "indices", "data"):
            assert bool((getattr(x.W, f) == getattr(y.W, f)).all())


def test_pyramid_round_trip(gsp):
    G = _random(gsp, 500, 21, np.float64)
    Gs, _ = gsp.reduction.tree_multiresolution(G, 3, root=0)
    f = np.random.default_rng(5).standard_normal(G.N)
    ca, pe = gsp.reduction.pyramid_analysis(Gs, f, order=30)
    rec, _ = gsp.reduction.pyramid_synthesis(Gs, ca[-1], pe, order=30)
    assert np.abs(rec[:, 0] - f).max() <= 1e-10


def test_compute_full_eigen(gsp):
    W = tro.random_tree(300, 4, decades=2)
    G = gsp.graphs.Graph(W, dtype=np.float64)
    Gs, _ = gsp.reduction.tree_multiresolution(G, 3, reduction_method="sum", root=2,
                                               compute_full_eigen=True)
    levels = tro.tree_multiresolution_levels(W, 3, "sum", 2)
    refs = [W] + [lev["W"] for lev in levels]
    for H, Wr in zip(Gs, refs):
        e_ref = np.linalg.eigvalsh(orc.laplacian(sparse.csr_matrix(Wr)).toarray())
        assert np.abs(np.asarray(H.e) - e_ref).max() <= 1e-10 * max(1.0, e_ref[-1])
