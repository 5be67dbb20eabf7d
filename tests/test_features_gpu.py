"""Graph features on the CUDA engine (pygsp_b200/features.py, csrc/moments.cu) against
tests/golden/features.npz, made by the unmodified PyGSP 0.6.1, and against the float64 oracle
(oracle/features_oracle.py) on graphs too large for the reference's frame."""
import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from, relerr_cols
from oracle import features_oracle as fo

pytestmark = pytest.mark.gpu

DTYPES = [np.float32, np.float64]
TOL = {np.float32: 2e-5, np.float64: 1e-10}


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def sensor_graph(gsp, z, dtype):
    G = gsp.graphs.Graph(csr_from(z, "sensor_W"), dtype=dtype)
    G._lmax = float(z["sensor_lmax"])
    G._lmax_method = "lanczos"
    return G


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_golden_parity(gsp, golden, dtype):
    z = golden("features")
    G = sensor_graph(gsp, z, dtype)
    lmax, tol = G.lmax, TOL[dtype]
    spectr = gsp.features.compute_spectrogram(G)
    assert isinstance(spectr, np.ndarray) and spectr.shape == (300, 100)
    assert spectr.dtype == np.float64 and G.spectr is spectr
    assert relerr_cols(spectr, z["spectr_default"]) <= tol
    spectr = gsp.features.compute_spectrogram(
        G, atom=lambda x: 1.0 / (1.0 + (10.0 * x / lmax) ** 2), M=20)
    assert spectr.shape == (300, 20)
    assert relerr_cols(spectr, z["spectr_atom"]) <= tol
    heat = gsp.features.compute_norm_tig(gsp.filters.Heat(G, scale=10))
    assert isinstance(heat, np.ndarray) and heat.shape == (300,)
    assert relerr_cols(heat, z["norm_heat"]) <= tol
    mh = gsp.features.compute_norm_tig(gsp.filters.MexicanHat(G, Nf=3))
    assert isinstance(mh, list) and len(mh) == 3
    for got, ref in zip(mh, z["norm_mh"]):
        assert got.shape == (900,)
        assert relerr_cols(got, ref) <= tol
    one = gsp.features.compute_norm_tig(gsp.filters.MexicanHat(G, Nf=3), i=1)
    assert one.shape == (900,)
    for g in ("sensor", "directed", "isolated"):
        Gw = gsp.graphs.Graph(csr_from(z, "adj_%s_W" % g), dtype=dtype)
        got = gsp.features.compute_avg_adj_deg(Gw)
        assert isinstance(got, np.ndarray) and got.dtype == np.float64
        np.testing.assert_array_equal(got, z["adj_" + g])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_moments_do_not_depend_on_chunking(gsp, golden, dtype):
    """A vertex's moments are the same bits at every width, at every position in its block."""
    import torch
    from pygsp_b200.filters.approximations import cheby_moments_device
    z = golden("features")
    G = sensor_graph(gsp, z, dtype)
    ref = cheby_moments_device(G.L, G.lmax, 30, width=64)
    assert ref.shape == (300, 61) and ref.dtype == torch.float64
    for width in (8, 128, 37, 300):
        assert torch.equal(cheby_moments_device(G.L, G.lmax, 30, width=width), ref), width
    mu = ref.cpu().numpy()
    np.testing.assert_array_equal(mu[:, 0], 1.0)
    L, lmax = G.L.to_scipy().astype(np.float64), G.lmax
    want = fo.moments(L, lmax, 30, np.arange(300))
    # float32 blocks: the recurrence's rounding grows with the order; 1.1e-5 measured at mu_60
    assert np.abs(mu - want).max() <= (1e-12 if dtype == np.float64 else 1e-4)


def test_large_morton_sensor(gsp):
    """2e4-vertex Morton Sensor graph, float32: 157 probe blocks of 128 columns (the tiled step),
    the last one partial; 64 sampled vertices against the float64 oracle."""
    import torch
    from pygsp_b200.filters.approximations import cheby_moments_device
    G = gsp.graphs.Sensor(20000, seed=7, order="morton", dtype=np.float32)
    G.estimate_lmax()
    assert G.L.tile_plan(128, 0) is not None and G.L.tile_plan(20000 % 128, 0) is not None
    lmax = G.lmax
    L = G.L.to_scipy().astype(np.float64)
    cols = np.sort(np.random.default_rng(3).choice(20000, 64, replace=False))
    cols[-1] = 19999                                 # a vertex of the partial last block
    spectr = gsp.features.compute_spectrogram(G)
    want = fo.square_norms_moments(L, lmax, fo.spectrogram_kernels(lmax), cols)
    assert relerr_cols(spectr[cols], want) <= TOL[np.float32]
    mu = cheby_moments_device(G.L, lmax, 30)
    assert torch.equal(mu[torch.as_tensor(cols, device=mu.device)],
                       cheby_moments_device(G.L, lmax, 30, width=64)[torch.as_tensor(cols, device=mu.device)])


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_order_50(gsp, golden, dtype):
    z = golden("features")
    G = sensor_graph(gsp, z, dtype)
    L = csr_from(z, "sensor_W")
    L = sparse.csgraph.laplacian(L).tocsr()
    f = gsp.filters.Heat(G, scale=10)
    got = gsp.features.compute_norm_tig(f, order=50)
    want = fo.norm_tig_frame(L, G.lmax, f._kernels, m=50)
    assert relerr_cols(got, want) <= TOL[dtype]
    assert relerr_cols(gsp.features.compute_norm_tig(f), z["norm_heat"]) <= TOL[dtype]


@pytest.mark.parametrize("dtype", DTYPES, ids=["f32", "f64"])
def test_exact_method(gsp, golden, dtype):
    z = golden("features")
    G = sensor_graph(gsp, z, dtype)
    G.compute_fourier_basis()
    U, e, lmax = G.U.astype(np.float64), G.e, G.lmax
    spectr = gsp.features.compute_spectrogram(G, method="exact")
    kern = fo.spectrogram_kernels(lmax)
    want = (U * U) @ np.stack([k(e) ** 2 for k in kern], axis=1)
    assert spectr.shape == (300, 100)
    assert relerr_cols(spectr, want) <= 1e-12
    f = gsp.filters.Heat(G, scale=10)
    got = gsp.features.compute_norm_tig(f, method="exact")
    assert relerr_cols(got, np.sqrt((U * U) @ (f._kernels[0](e) ** 2))) <= 1e-12
    # order 30 is close to exact for the smooth heat kernel
    assert relerr_cols(gsp.features.compute_norm_tig(f), got) <= 1e-4


def test_compute_tig_is_the_frame(gsp, golden):
    z = golden("features")
    G = sensor_graph(gsp, z, np.float64)
    f = gsp.filters.MexicanHat(G, Nf=3)
    tig = gsp.features.compute_tig(f)
    assert isinstance(tig, list) and len(tig) == 3
    frame = f.compute_frame()
    for t in tig:
        np.testing.assert_array_equal(t, frame)
    assert relerr_cols(np.linalg.norm(frame, axis=1), z["norm_mh"][0]) <= 1e-10


def _boolean_reference(W):
    return fo.avg_adj_deg(W)


def test_avg_adj_deg_large(gsp):
    """1e5-vertex k-NN graph (light rows) and the same graph with a 3000-neighbour hub."""
    G = gsp.graphs.Sensor(100000, seed=1, dtype=np.float32)
    W = G.W.to_scipy()
    np.testing.assert_array_equal(gsp.features.compute_avg_adj_deg(G), _boolean_reference(W))
    hub = np.random.default_rng(2).choice(np.arange(1, 100000), 3000, replace=False)
    H = sparse.lil_matrix(W)
    H[0, hub] = 1.0
    H[hub, 0] = 1.0
    H = sparse.csr_matrix(H)
    Gh = gsp.graphs.Graph(H, dtype=np.float64)
    np.testing.assert_array_equal(gsp.features.compute_avg_adj_deg(Gh), _boolean_reference(H))


def test_avg_adj_deg_star(gsp):
    """A 5000-leaf star: every row is heavy (5000 candidates), several chunks of hash tables."""
    n = 5001
    rows = np.r_[np.zeros(n - 1, dtype=int), np.arange(1, n)]
    cols = np.r_[np.arange(1, n), np.zeros(n - 1, dtype=int)]
    W = sparse.csr_matrix((np.ones(2 * (n - 1)), (rows, cols)), shape=(n, n))
    G = gsp.graphs.Graph(W, dtype=np.float32)
    got = gsp.features.compute_avg_adj_deg(G)
    want = _boolean_reference(W)
    np.testing.assert_array_equal(got, want)
    assert got[0, 0] == 1.0 / n and got[1, 0] == (n - 1) / 2.0
