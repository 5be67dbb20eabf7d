"""GPU parity tests: the CUDA path (through the C ABI) against the oracle and the
golden fixtures generated from PyGSP 0.6.1.  Run on an H100: pytest -m gpu.

Tolerances (BASELINE.json north_star / SURVEY.md 8c):
  * CSR indptr / indices of L: bit-exact;
  * values of L: 1e-6 relative (float32 engine), 1e-12 (float64 engine);
  * filter outputs: per column max|y - ref| / max|ref| <= 1e-5 (float32 engine),
    <= 1e-10 (float64 engine; the reference's own tests use 1e-7 .. 1e-10).
"""
import numpy as np
import pytest

from conftest import csr_from, relerr_cols
from oracle import pygsp_oracle as orc

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5
F64_TOL = 1e-10


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def _tol(dtype):
    return F32_TOL if np.dtype(dtype) == np.float32 else F64_TOL


def _fix_lmax(G, lmax):
    G._lmax = float(lmax)
    G._lmax_method = "lanczos"


# --------------------------------------------------------------------- Laplacian
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_laplacian_kats(gsp, golden, dtype):
    g = golden("laplacian_kat")
    vtol = 1e-12 if dtype == np.float64 else 2e-6
    for name in g["names"]:
        A = g[name + "_A"]
        for lap in ("combinatorial", "normalized"):
            G = gsp.graphs.Graph(A, lap_type=lap, dtype=dtype)
            ref = csr_from(g, name + "_L" + lap[0])
            L = G.L.to_scipy()
            np.testing.assert_array_equal(L.indptr, ref.indptr, err_msg=name + lap)
            np.testing.assert_array_equal(L.indices, ref.indices, err_msg=name + lap)
            np.testing.assert_allclose(L.data, ref.data, rtol=vtol, atol=0, err_msg=name + lap)
            assert L.indptr.dtype == np.int32 and L.indices.dtype == np.int32
            assert G.is_directed() == bool(g[name + "_directed"])
            assert G.n_edges == int(g[name + "_n_edges"]) == G.Ne
            np.testing.assert_allclose(G.dw, g[name + "_dw"], rtol=vtol)
            np.testing.assert_allclose(G.d, g[name + "_d"])
            ref_bound = float(g[name + "_bound_" + lap[0]])
            got = G._get_upper_bound()
            if np.isnan(ref_bound):
                assert np.isnan(got)
            else:
                np.testing.assert_allclose(got, ref_bound, rtol=max(vtol, 1e-12), err_msg=name)


@pytest.mark.parametrize("fixture,prefix", [("logo", "logo"), ("sensor123", "s"), ("grid13x9", "g")])
def test_laplacian_fixtures(gsp, golden, fixture, prefix):
    g = golden(fixture)
    W = csr_from(g, "W")
    for dtype, vtol in ((np.float64, 1e-12), (np.float32, 2e-6)):
        G = gsp.graphs.Graph(W, dtype=dtype)
        for lap in ("combinatorial", "normalized"):
            G.compute_laplacian(lap)
            ref = csr_from(g, prefix + "_L" + lap[0])
            L = G.L.to_scipy()
            np.testing.assert_array_equal(L.indptr, ref.indptr)
            np.testing.assert_array_equal(L.indices, ref.indices)
            np.testing.assert_allclose(L.data, ref.data, rtol=vtol, atol=0)
            np.testing.assert_allclose(G._get_upper_bound(), float(g[prefix + "_bound_" + lap[0]]),
                                       rtol=max(vtol, 1e-12))


def test_adjacency_formats_and_checks(gsp, golden, caplog):
    """pygsp/tests/test_graphs.py:464-485 (dtype/format matrix), :432-461 (empty graph)."""
    from scipy import sparse
    g = golden("sensor123")
    W = csr_from(g, "W")
    ref = csr_from(g, "s_Lc")
    for conv in (sparse.csr_matrix, sparse.csc_matrix, sparse.coo_matrix, sparse.lil_matrix,
                 lambda m: m.toarray(), lambda m: m.astype(np.float32)):
        L = gsp.graphs.Graph(conv(W), dtype=np.float64).L.to_scipy()
        np.testing.assert_array_equal(L.indices, ref.indices)
        np.testing.assert_allclose(L.data, ref.data, rtol=1e-6)
    Wi = (W > 0).astype(np.int64)                     # integer / boolean adjacency
    G = gsp.graphs.Graph(Wi, dtype=np.float64)
    assert G.L.nnz == ref.nnz
    G = gsp.graphs.Graph(np.zeros((6, 6)))
    assert G.n_edges == 0 and G.L.nnz == 0 and G.W.nnz == 0
    # explicit zeros are eliminated; duplicates of a COO input are summed
    coo = sparse.coo_matrix(([1.0, 2.0, 0.0, 3.0, 3.0], ([0, 0, 1, 1, 2], [1, 1, 2, 0, 2])), shape=(3, 3))
    G = gsp.graphs.Graph(coo, dtype=np.float64)
    assert G.W.nnz == 3 and G.has_loops()
    np.testing.assert_allclose(G.W.toarray(), [[0, 3, 0], [3, 0, 0], [0, 0, 3]])
    with pytest.raises(ValueError):
        gsp.graphs.Graph(np.ones((3, 4)))
    with pytest.raises(ValueError):
        gsp.graphs.Graph([[0, np.nan], [1, 0]])
    with pytest.raises(ValueError):
        gsp.graphs.Graph([[0, np.inf], [1, 0]])
    with pytest.raises(ValueError):
        gsp.graphs.Graph(np.zeros((3, 3)), lap_type="unknown")
    with pytest.raises(AttributeError):
        G.W = W
    with pytest.raises(AttributeError):
        G.lmax = 3.0


# ---------------------------------------------------------------------------- lmax
def test_lmax_kats(gsp):
    """pygsp/tests/test_graphs.py:257-294: graphs whose algebraic bound is tight."""
    cases = [(np.full((10, 10), 2), "combinatorial", 20.0),
             ([[0, 0, 1, 1], [0, 0, 1, 1], [1, 1, 0, 0], [1, 1, 0, 0]], "combinatorial", 4.0),
             ([[0, 0, 1, 1], [0, 0, 1, 0], [1, 1, 0, 0], [1, 0, 0, 0]], "normalized", 2.0)]
    for A, lap, lmax in cases:
        for dtype, rtol in ((np.float64, 1e-7), (np.float32, 1e-5)):
            G = gsp.graphs.Graph(A, lap_type=lap, dtype=dtype)
            G.estimate_lmax(method="bounds")
            np.testing.assert_allclose(G.lmax, lmax, rtol=rtol)
            G.estimate_lmax(method="lanczos")
            np.testing.assert_allclose(G.lmax, lmax * 1.01, rtol=rtol)
    G = gsp.graphs.Graph(cases[1][0])
    with pytest.raises(ValueError):
        G.estimate_lmax(method="unk")


def test_lmax_logo_and_laziness(gsp, golden, caplog):
    g = golden("logo")
    for dtype in (np.float64, np.float32):
        G = gsp.graphs.Logo(dtype=dtype)
        lo, hi = orc.lmax_lanczos_band(csr_from(g, "logo_Lc"))
        G.estimate_lmax()
        assert lo <= G.lmax <= hi * (1 + 1e-5), (lo, G.lmax, hi)
        assert "{:.2f}".format(G.lmax) == "13.92"               # graph.py:891-899
        first = G.lmax
        G.estimate_lmax()                                       # cached: no-op
        assert G.lmax == first
        G.estimate_lmax(method="bounds")
        assert "{:.2f}".format(G.lmax) == "18.58"
        # changing the Laplacian invalidates lmax; the lazy property warns and re-estimates
        G.compute_laplacian("normalized")
        with caplog.at_level("WARNING"):
            assert 0 < G.lmax <= 2 * 1.01
        assert any("G.lmax is not available" in r.getMessage() for r in caplog.records)
    # reproducible: same seed, same value (the reference's ARPACK start vector is unseeded)
    a = gsp.graphs.Logo(); a.estimate_lmax()
    b = gsp.graphs.Logo(); b.estimate_lmax()
    assert a.lmax == b.lmax


# ---------------------------------------------------------------- filtering: goldens
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_readme_example(gsp, golden, dtype):
    """README.rst:68-89 == BASELINE config 1."""
    g = golden("logo")
    G = gsp.graphs.Logo(dtype=dtype)
    _fix_lmax(G, g["lmax_lanczos"])
    h = gsp.filters.Heat(G, scale=50)
    c = gsp.filters.compute_cheby_coeff(h, m=30)
    np.testing.assert_allclose(c, g["heat50_coeff"], rtol=1e-10, atol=1e-14)
    y = h.filter(g["readme_signal"])
    assert isinstance(y, np.ndarray) and y.shape == (G.N,)
    assert relerr_cols(y, g["readme_filtered"]) <= _tol(dtype)
    r = gsp.filters.cheby_rect(G, [2.0, 6.0], g["rect_signal"], order=25)
    assert relerr_cols(r, g["rect_filtered"]) <= _tol(dtype)
    with pytest.raises(ValueError):
        gsp.filters.cheby_rect(G, [1.0], g["rect_signal"])


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_sensor123_goldens(gsp, golden, dtype):
    g = golden("sensor123")
    tol = _tol(dtype)
    G = gsp.graphs.Graph(csr_from(g, "W"), dtype=dtype)
    _fix_lmax(G, g["lmax"])
    h = gsp.filters.Heat(G)
    y = h.filter(g["signal"], method="chebyshev")
    assert relerr_cols(y, g["heat10_cheb"]) <= tol
    if dtype == np.float64:                                  # test_filters.py:403-417
        np.testing.assert_allclose(y, g["heat10_exact"], rtol=1e-7)
    with pytest.raises(ValueError):
        h.filter(g["signal"], method="lanczos")
    # frame of Heat([8, 9]) by filtering the identity (test_filters.py:157-168)
    h89 = gsp.filters.Heat(G, scale=[8, 9])
    F = gsp.filters.cheby_op(G, gsp.filters.compute_cheby_coeff(h89, m=30), np.identity(G.N))
    assert F.shape == (2 * G.N, G.N)
    assert relerr_cols(F, g["heat89_frame"]) <= tol
    if dtype == np.float64:
        np.testing.assert_allclose(F, g["heat89_frame"], atol=1e-10)
    F2 = h89.compute_frame(method="chebyshev", order=30)      # filter.py:540-603
    assert F2.shape == (2 * G.N, G.N) and relerr_cols(F2, g["heat89_frame"]) <= tol
    mh = gsp.filters.MexicanHat(G, Nf=5)
    c = np.array(gsp.filters.compute_cheby_coeff(mh, m=40))
    np.testing.assert_allclose(c, g["mh5_coeff"], rtol=1e-10, atol=1e-13)
    assert relerr_cols(gsp.filters.cheby_op(G, c, g["mh5_block"]), g["mh5_cheby_op"]) <= tol
    a = mh.filter(g["mh5_block"], order=40)
    assert a.shape == (G.N, 3, 5)
    assert relerr_cols(a, g["mh5_analysis"]) <= tol
    s = mh.filter(g["mh5_analysis"], order=40)
    assert s.shape == (G.N, 3)
    assert relerr_cols(s, g["mh5_synthesis"]) <= tol
    assert relerr_cols(mh.synthesize(mh.analyze(g["mh5_block"], order=40), order=40),
                       g["mh5_synthesis"]) <= 10 * tol
    assert relerr_cols(h.localize(7, order=25), g["localize_7"]) <= tol


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_shape_truth_table(gsp, golden, dtype):
    """filter.py:267-290,328 -- SURVEY.md 3.5; test_filters.py:87-122."""
    import torch
    g = golden("sensor123")
    tol = _tol(dtype)
    G = gsp.graphs.Graph(csr_from(g, "W"), dtype=dtype)
    _fix_lmax(G, g["lmax"])
    mh = gsp.filters.MexicanHat(G, Nf=5)
    heat = gsp.filters.Heat(G, 10)
    for j in range(9):
        x = g["tt%d_in" % j]
        y = mh.filter(x, order=20)
        assert y.shape == g["tt%d_mh5" % j].shape, x.shape
        assert relerr_cols(y, g["tt%d_mh5" % j]) <= tol
        yt = mh.filter(torch.from_numpy(x).cuda(), order=20)      # device in -> device out
        assert yt.is_cuda and tuple(yt.shape) == y.shape
        np.testing.assert_array_equal(yt.cpu().numpy(), y)
        if "tt%d_heat" % j in g:
            y = heat.filter(x, order=20)
            assert y.shape == g["tt%d_heat" % j].shape
            assert relerr_cols(y, g["tt%d_heat" % j]) <= tol
    n = G.N
    with pytest.raises(ValueError):
        mh.filter(np.zeros((n, 3, 2)))
    with pytest.raises(ValueError):
        mh.filter(np.zeros((n, 3, 1, 1)))
    with pytest.raises(ValueError):
        mh.filter(np.zeros(n + 1))
    with pytest.raises(TypeError):
        heat.filter(np.zeros(n), order=0)
    with pytest.raises(TypeError):
        gsp.filters.cheby_op(G, [1.0], np.zeros(n))
    with pytest.raises(ValueError):
        mh.analyze(np.zeros((n, 3, 5)))
    with pytest.raises(ValueError):
        mh.synthesize(np.zeros((n, 3, 4)))
    assert heat.filter(np.ones(n), order=1).shape == (n,)
    assert heat.filter(list(range(n))).shape == (n,)             # lists / ints accepted
    x = g["tt3_in"].copy()
    heat.filter(x)
    np.testing.assert_array_equal(x, g["tt3_in"])                # inputs are never mutated
    assert (heat @ x).shape == heat.filter(x).shape
    assert len(mh) == 5 and mh[1:3].Nf == 2 and (mh + heat).Nf == 6
    assert mh.evaluate(np.linspace(0, G.lmax, 7)).shape == (5, 7)


def test_doctest_goldens(gsp, golden):
    """filter.py:217-219 and :232-256 (0.27649)."""
    g = golden("doctest")
    for dtype in (np.float64, np.float32):
        G = gsp.graphs.Graph(csr_from(g, "W"), dtype=dtype)
        _fix_lmax(G, g["lmax"])
        s1 = np.zeros(G.N); s1[13] = 1
        s1 = gsp.filters.Heat(G, 3).filter(s1)
        assert s1.shape == (30,)
        mh = gsp.filters.MexicanHat(G, Nf=4)
        s2 = mh.analyze(s1)
        assert s2.shape == (30, 4)
        s3 = mh.synthesize(s2)
        assert s3.shape == (30,)
        if dtype == np.float64:
            assert "{:.5f}".format(np.linalg.norm(s1 - s3)) == "0.27649"
        assert abs(np.linalg.norm(s1 - s3) - float(g["norm"])) < 1e-5
        R = gsp.graphs.Graph(csr_from(g, "ringW"), dtype=dtype)
        _fix_lmax(R, g["ring_lmax"])
        y = gsp.filters.Heat(R, [1, 10, 100]).filter(g["ring_signal"])
        assert y.shape == (60, 10, 3)
        assert relerr_cols(y, g["ring_filtered"]) <= _tol(dtype)


def test_grid_bank_golden(gsp, golden):
    g = golden("grid13x9")
    for dtype in (np.float64, np.float32):
        G = gsp.graphs.Grid2d(13, 9, dtype=dtype)
        np.testing.assert_array_equal(G.L.to_scipy().indices, csr_from(g, "g_Lc").indices)
        _fix_lmax(G, g["lmax"])
        y = gsp.filters.MexicanHat(G, Nf=6).filter(g["signal"], order=50)
        assert relerr_cols(y, g["filtered"]) <= _tol(dtype)


# ------------------------------------------------- filtering: oracle on seeded inputs
@pytest.fixture(scope="module")
def sensor5k(gsp):
    rng = np.random.default_rng(5)
    G = gsp.graphs.Sensor(5000, k=8, seed=11, order="morton", dtype=np.float32)
    G.estimate_lmax()
    L = orc.laplacian(G.W.to_scipy().astype(np.float64))
    return G, L, rng


@pytest.mark.parametrize("nsig", [1, 2, 3, 4, 5, 8, 12, 16, 31, 32, 33, 64, 96, 128, 132, 200])
def test_cheby_op_signal_widths(gsp, sensor5k, nsig):
    G, L, _ = sensor5k
    rng = np.random.default_rng(nsig)
    x = rng.standard_normal((G.N, nsig))
    c = orc.cheby_coeff(orc.heat_kernels(G.lmax, 30), G.lmax, 24)
    ref = orc.cheby_op(L, G.lmax, c, x)
    y = gsp.filters.cheby_op(G, c, x.astype(np.float32))
    assert y.dtype == np.float32 and y.shape == ref.shape
    assert relerr_cols(y, ref) <= F32_TOL


@pytest.mark.parametrize("nscales,nsig", [(1, 64), (2, 8), (6, 64), (6, 3), (17, 4), (33, 1)])
def test_cheby_op_filter_banks(gsp, sensor5k, nscales, nsig):
    """Banks of 1 to 33 filters through the public cheby_op: up to 16 the fused step, wider
    banks the stored-basis route (cheby_bank_device).  The fused step's axpy path for more than
    16 scales (cheby_axpy_scales) is tested directly in test_filter_banks_gpu.py."""
    G, L, _ = sensor5k
    rng = np.random.default_rng(1000 + nscales)
    x = rng.standard_normal((G.N, nsig))
    c = rng.standard_normal((nscales, 21)) / np.arange(1, 22) ** 2
    ref = orc.cheby_op(L, G.lmax, c, x)
    y = gsp.filters.cheby_op(G, c, x.astype(np.float32))
    assert relerr_cols(y, ref) <= F32_TOL


def test_cheby_op_edge_graphs(gsp):
    """Isolated vertices (empty Laplacian rows), a hub row far longer than a lane
    group, unaligned views, order 1, float64 engine."""
    import torch
    from scipy import sparse
    rng = np.random.default_rng(9)
    n = 700
    A = sparse.random(n, n, 0.01, random_state=9, format="lil")
    A[0, :] = rng.uniform(size=n) * (rng.uniform(size=n) < 0.9)     # hub: ~630 neighbours
    A = sparse.csr_matrix(A)
    A = A + A.T
    A.setdiag(0)
    A = A.tolil()
    A[5, :] = 0; A[:, 5] = 0; A[6, :] = 0; A[:, 6] = 0              # isolated vertices
    A = sparse.csr_matrix(A)
    A.eliminate_zeros()
    for dtype in (np.float32, np.float64):
        G = gsp.graphs.Graph(A, dtype=dtype)
        assert G.L.to_scipy().indptr[6] == G.L.to_scipy().indptr[5]
        G.estimate_lmax()
        L = orc.laplacian(A)
        np.testing.assert_array_equal(G.L.to_scipy().indices, L.indices)
        for nsig, order in ((7, 30), (64, 1), (1, 12)):
            x = rng.standard_normal((n, nsig))
            c = orc.cheby_coeff(orc.heat_kernels(G.lmax, [5, 40]), G.lmax, order)
            ref = orc.cheby_op(L, G.lmax, c, x)
            y = gsp.filters.cheby_op(G, c, x)
            assert relerr_cols(y, ref) <= _tol(dtype)
        # isolated vertex: T_1 = -x, output = p(0) x
        x = rng.standard_normal(n)
        y = gsp.filters.Heat(G, 10).filter(x)
        assert abs(y[5] / x[5] - 1) < 1e-4
    # a non-contiguous / offset device view is made contiguous, not misread
    G = gsp.graphs.Graph(A)
    G.estimate_lmax()
    big = torch.randn(n, 9, device="cuda")
    view = big[:, 1:8:2]
    y = gsp.filters.Heat(G, 10).filter(view)
    y2 = gsp.filters.Heat(G, 10).filter(view.contiguous())
    assert torch.equal(y, y2)


def test_lmax_brackets_truth(gsp, sensor5k):
    G, L, _ = sensor5k
    lam = orc.lambda_max_exact(L)
    assert lam * (1 - 1e-4) <= G.lmax / 1.01 <= lam * (1 + 1e-5)
    G64 = gsp.graphs.Graph(G.W.to_scipy(), dtype=np.float64)
    G64.estimate_lmax()
    assert lam * (1 - 1e-4) <= G64.lmax / 1.01 <= lam * (1 + 1e-9)


@pytest.mark.parametrize("nsig,order", [(64, 30), (64, 1), (64, 2), (64, 3), (32, 17), (5, 12), (128, 8)])
def test_clenshaw_matches_forward_recurrence(gsp, sensor5k, nsig, order):
    """SURVEY.md 8f rank 1: Clenshaw evaluation of the same Chebyshev sum."""
    G, L, _ = sensor5k
    rng = np.random.default_rng(order * 100 + nsig)
    x = rng.standard_normal((G.N, nsig))
    c = orc.cheby_coeff(orc.heat_kernels(G.lmax, 20), G.lmax, order)
    ref = orc.cheby_op(L, G.lmax, c, x)
    y = gsp.filters.cheby_op(G, c, x.astype(np.float32), clenshaw=True)
    assert y.shape == ref.shape and relerr_cols(y, ref) <= F32_TOL
    G64 = gsp.graphs.Graph(G.W.to_scipy(), dtype=np.float64)
    G64._lmax, G64._lmax_method = G.lmax, "lanczos"
    assert relerr_cols(gsp.filters.cheby_op(G64, c, x, clenshaw=True), ref) <= F64_TOL
    with pytest.raises(ValueError):
        gsp.filters.cheby_op(G, np.vstack([c, c]), x, clenshaw=True)


def test_heavy_rows_fall_back_to_rowgroup(gsp):
    """A hub whose CSR slab cannot fit a shared-memory stage: the tile plan declines and
    the row-group kernel serves the whole matrix (same results, float32 Nsig=64)."""
    from scipy import sparse
    n = 70000
    rng = np.random.default_rng(4)
    hub = np.zeros(n - 1, dtype=np.int64)
    ring = np.arange(1, n)
    rows = np.concatenate([hub, ring[:-1]])
    cols = np.concatenate([ring, ring[1:]])
    w = rng.uniform(0.5, 1.5, rows.size)
    A = sparse.coo_matrix((w, (rows, cols)), shape=(n, n)).tocsr()
    A = A + A.T
    G = gsp.graphs.Graph(A)
    assert G.L.tile_plan(64, 1) is None                   # 70 000-entry row: no tiling
    G.estimate_lmax(method="bounds")
    L = orc.laplacian(A)
    x = rng.standard_normal((n, 64))
    c = orc.cheby_coeff(orc.heat_kernels(G.lmax, 30), G.lmax, 10)
    assert relerr_cols(gsp.filters.cheby_op(G, c, x), orc.cheby_op(L, G.lmax, c, x)) <= F32_TOL


def test_normalized_and_directed_graphs_filter(gsp, golden):
    """lap_type='normalized' and a directed adjacency go through the same filter path."""
    from scipy import sparse
    rng = np.random.default_rng(8)
    A = sparse.random(3000, 3000, 0.002, random_state=8, format="csr")       # directed
    A.setdiag(0); A.eliminate_zeros()
    x = rng.standard_normal((3000, 32))
    for lap in ("combinatorial", "normalized"):
        G = gsp.graphs.Graph(A, lap_type=lap)
        assert G.is_directed()
        L = orc.laplacian(A, lap)
        Ld = G.L.to_scipy()
        np.testing.assert_array_equal(Ld.indptr, L.indptr)
        np.testing.assert_array_equal(Ld.indices, L.indices)
        np.testing.assert_allclose(Ld.data, L.data, rtol=3e-6, atol=1e-7)
        G.estimate_lmax()
        c = orc.cheby_coeff(orc.mexican_hat_kernels(G.lmax, Nf=3), G.lmax, 20)
        # the oracle takes the device's float32 Laplacian values so that only the
        # recurrence is compared
        ref = orc.cheby_op(Ld.astype(np.float64), G.lmax, c, x)
        assert relerr_cols(gsp.filters.cheby_op(G, c, x), ref) <= F32_TOL


@pytest.mark.parametrize("nf,nsig,order", [(5, 64, 30), (2, 32, 12), (6, 3, 20), (3, 64, 1), (16, 8, 9)])
def test_fused_synthesis_matches_reference_order(gsp, sensor5k, nf, nsig, order):
    """SURVEY.md 8f rank 2: synthesis as one backward recurrence == sum of forward ones."""
    G, L, _ = sensor5k
    rng = np.random.default_rng(nf * 1000 + nsig)
    s = rng.standard_normal((G.N, nsig, nf))
    bank = gsp.filters.Heat(G, scale=[3.0 * (i + 1) for i in range(nf)])
    ref = orc.filter_signal(L, G.lmax, orc.heat_kernels(G.lmax, bank.scale), s, order=order)
    assert bank.fused_synthesis
    y = bank.filter(s.astype(np.float32), order=order)
    assert y.shape == ref.shape and relerr_cols(y, ref) <= F32_TOL
    bank.fused_synthesis = False                        # the reference's operation order
    y2 = bank.filter(s.astype(np.float32), order=order)
    assert relerr_cols(y2, ref) <= F32_TOL
    G64 = gsp.graphs.Graph(G.W.to_scipy(), dtype=np.float64)
    G64._lmax, G64._lmax_method = G.lmax, "lanczos"
    b64 = gsp.filters.Heat(G64, scale=bank.scale)
    assert relerr_cols(b64.filter(s, order=order), ref) <= F64_TOL


@pytest.mark.parametrize("n,dim,k", [(20000, 2, 10), (6000, 3, 16), (500, 2, 32), (40, 2, 3)])
def test_device_knn_equals_kdtree(gsp, n, dim, k):
    """SURVEY.md 8f-4: grid-hash k-NN on the GPU vs scipy.spatial.cKDTree (nngraph.py:213-216)."""
    from scipy import spatial
    pts = np.random.default_rng(n + dim).uniform(size=(n, dim))
    if n == 500:
        pts[:, 0] *= 7.0                                   # anisotropic box
    D, NN = spatial.cKDTree(pts).query(pts, k=k + 1)
    nn, dist = gsp.graphs.knn_device(pts, k)
    np.testing.assert_array_equal(nn.cpu().numpy(), NN[:, 1:])
    np.testing.assert_allclose(dist.cpu().numpy(), D[:, 1:], rtol=1e-12, atol=1e-15)


def test_device_generators_equal_host_generators(gsp):
    """Sensor / NNGraph / Grid2d built in HBM give the same adjacency as the host builders."""
    for kw in (dict(N=30000, k=10, seed=3, order="morton"), dict(N=2000, k=6, seed=1)):
        H = gsp.graphs.Sensor(backend="host", dtype=np.float64, **kw)
        D = gsp.graphs.Sensor(backend="device", dtype=np.float64, **kw)
        Wh, Wd = H.W.to_scipy(), D.W.to_scipy()
        np.testing.assert_array_equal(Wd.indptr, Wh.indptr)
        np.testing.assert_array_equal(Wd.indices, Wh.indices)
        np.testing.assert_allclose(Wd.data, Wh.data, rtol=1e-12)
        assert abs(D.sigma - H.sigma) <= 1e-13 * H.sigma and D.n_edges == H.n_edges
        np.testing.assert_array_equal(D.L.to_scipy().indices, H.L.to_scipy().indices)
    pts = np.random.default_rng(0).normal(size=(5000, 3))
    H = gsp.graphs.NNGraph(pts, k=8, backend="host", dtype=np.float64)
    D = gsp.graphs.NNGraph(pts, k=8, backend="device", dtype=np.float64)
    np.testing.assert_array_equal(D.W.to_scipy().indices, H.W.to_scipy().indices)
    np.testing.assert_allclose(D.W.to_scipy().data, H.W.to_scipy().data, rtol=1e-11)
    for shape in ((7, 5), (1, 9), (64, 64)):
        H = gsp.graphs.Grid2d(*shape, backend="host")
        D = gsp.graphs.Grid2d(*shape, backend="device")
        np.testing.assert_array_equal(D.W.to_scipy().indptr, H.W.to_scipy().indptr)
        np.testing.assert_array_equal(D.W.to_scipy().indices, H.W.to_scipy().indices)
        np.testing.assert_array_equal(D.W.to_scipy().data, H.W.to_scipy().data)
        assert D.n_edges == H.n_edges


def test_arbitrary_kernel_high_order(gsp, sensor5k):
    """Any kernel function plugs into Filter: the Green kernel 1/(eps + x) at order 100 is
    what reduction.interpolate feeds to the same path (reduction.py:150-193)."""
    G, L, _ = sensor5k
    green = lambda x: 1.0 / (0.05 + x)
    x = np.random.default_rng(3).standard_normal((G.N, 16))
    y = gsp.filters.Filter(G, green).filter(x.astype(np.float32), order=100)
    ref = orc.filter_signal(L, G.lmax, [green], x, order=100)
    assert relerr_cols(y, ref) <= F32_TOL


def test_graph_from_device_coo(gsp):
    """COO -> CSR on the device == scipy.sparse.csr_matrix(coo) (graph.py:109)."""
    import torch
    from scipy import sparse
    rng = np.random.default_rng(12)
    n, m = 3000, 40000
    r = rng.integers(0, n, m); c = rng.integers(0, n, m)
    keep = r != c
    r, c = r[keep], c[keep]
    v = rng.uniform(0.1, 1.0, r.size)
    rows = np.concatenate([r, c]); cols = np.concatenate([c, r]); vals = np.concatenate([v, v])
    ref = sparse.csr_matrix(sparse.coo_matrix((vals, (rows, cols)), shape=(n, n)))   # sums duplicates
    G = gsp.graphs.Graph.from_coo(torch.from_numpy(rows).cuda(), torch.from_numpy(cols).cuda(),
                                  torch.from_numpy(vals).cuda(), n, dtype=np.float64)
    W = G.W.to_scipy()
    np.testing.assert_array_equal(W.indptr, ref.indptr)
    np.testing.assert_array_equal(W.indices, ref.indices)
    np.testing.assert_allclose(W.data, ref.data, rtol=1e-13)
    assert not G.is_directed()
    L = orc.laplacian(ref)
    np.testing.assert_array_equal(G.L.to_scipy().indices, L.indices)
    with pytest.raises(gsp._native.NativeError):
        gsp.graphs.Graph.from_coo(torch.tensor([0, 5]).cuda(), torch.tensor([1, 0]).cuda(),
                                  torch.tensor([1.0, 1.0]).cuda(), 3)


def test_spmm_dot(gsp, sensor5k):
    G, L, _ = sensor5k
    x = np.random.default_rng(2).standard_normal((G.N, 10))
    y = G.L.dot(x)
    assert relerr_cols(y, L.dot(x)) <= F32_TOL
    assert relerr_cols(G.L.dot(x[:, 0]), L.dot(x[:, 0])) <= F32_TOL


# ---------------------------------------- full size: size-independent properties
@pytest.fixture(scope="module")
def sensor1m(gsp):
    G = gsp.graphs.Sensor(1_000_000, k=10, seed=0, order="morton")
    G.estimate_lmax()
    return G


def test_full_size_properties(gsp, sensor1m):
    """BASELINE config 2 (N=1e6, k=10, 64 signals, Heat(50), order 30)."""
    import torch
    G = sensor1m
    assert G.L.nnz == G.W.nnz + G.N                  # connected-degree diagonal everywhere
    L = G.L.to_scipy()
    assert L.has_canonical_format
    assert abs(L.sum(axis=1)).max() < 1e-3           # rows of a combinatorial Laplacian sum to 0
    h = gsp.filters.Heat(G, scale=50)
    c = gsp.filters.compute_cheby_coeff(h, m=30)
    gen = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(G.N, 64, device="cuda", generator=gen)
    y = h.filter(x, order=30)
    assert y.shape == (G.N, 64) and bool(torch.isfinite(y).all())
    # (1) constants are eigenvectors for eigenvalue 0: output = p(0) * input
    p0 = 0.5 * c[0] + sum(c[k] * (-1) ** k for k in range(1, 31))
    ones = torch.ones(G.N, 4, device="cuda")
    yc = h.filter(ones, order=30)
    assert float((yc - p0).abs().max()) <= 2e-5 * abs(p0)
    # (2) linearity
    a, b = 0.75, -1.5
    z = torch.randn(G.N, 64, device="cuda", generator=gen)
    lhs = h.filter(a * x + b * z, order=30)
    rhs = a * y + b * h.filter(z, order=30)
    assert float((lhs - rhs).abs().max() / rhs.abs().max()) <= 1e-5
    # (3) columns are independent: filtering a column alone gives the same bits
    y7 = h.filter(x[:, 7].contiguous(), order=30)
    assert float((y7 - y[:, 7]).abs().max() / y7.abs().max()) <= 2e-6
    # (4) two columns against the float64 oracle at full size
    Lo = L.astype(np.float64)
    ref = orc.cheby_op(Lo, G.lmax, c, x[:, :2].double().cpu().numpy())
    assert relerr_cols(y[:, :2].cpu().numpy(), ref) <= F32_TOL
    # (5) lmax respects the algebraic bound and dominates the Rayleigh quotient of y
    assert G.lmax <= 1.01 * G._get_upper_bound() * (1 + 1e-5)
    v = torch.randn(G.N, 1, device="cuda", generator=gen)
    for _ in range(20):
        v = G.L.dot(v)
        v = v / v.norm()
    rq = float((v * G.L.dot(v)).sum())
    assert rq <= G.lmax / 1.01 * (1 + 1e-4) and G.lmax <= 1.01 * rq * 1.2


# ---------------------------------------------------------- round 2: SpMV, pipeline
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_spmv_subwarp_matches_scipy(gsp, dtype):
    """gsp_spmv_* (sub-warp rows, shuffle reduction) on graphs of very different mean degree."""
    import torch
    from scipy import sparse
    rng = np.random.default_rng(5)
    mats = [gsp.graphs.Sensor(3000, k=10, seed=1, dtype=dtype).L.to_scipy(),
            gsp.graphs.Grid2d(37, 41, dtype=dtype).L.to_scipy(),
            sparse.random(500, 500, 0.3, random_state=3, format="csr", dtype=np.float64),
            sparse.random(400, 400, 0.004, random_state=4, format="csr", dtype=np.float64),
            sparse.csr_matrix((7, 7), dtype=np.float64)]
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    for M in mats:
        M = M.astype(np.float64).tocsr()
        M.sort_indices()
        D = gsp.graphs.DeviceCSR.from_scipy(M, tdt, torch.device("cuda"))
        v = rng.standard_normal(M.shape[1])
        got = D.dot(v)
        ref = M.dot(v)
        assert got.shape == ref.shape
        scale = max(np.abs(ref).max(), 1e-30)
        assert np.abs(got - ref).max() / scale <= (2e-6 if dtype == np.float32 else 1e-13)


def test_staging_copies_move_column_chunks(gsp):
    """gsp_copy2d_async and gsp_stage_cols: a strided column chunk host -> device -> host."""
    import ctypes
    import torch
    from pygsp_b200 import _native as nat
    n, nsig, w = 1000, 64, 16
    xh = torch.randn(n, nsig).pin_memory()
    for use_kernel in (False, True):
        dev = torch.zeros(n, w, device="cuda")
        back = torch.zeros(n, nsig).pin_memory()
        st = torch.cuda.current_stream()
        for j in range(nsig // w):
            args_in = (ctypes.c_void_p(dev.data_ptr()), ctypes.c_size_t(w * 4),
                       ctypes.c_void_p(xh.data_ptr() + j * w * 4), ctypes.c_size_t(nsig * 4),
                       ctypes.c_size_t(w * 4), ctypes.c_size_t(n))
            args_out = (ctypes.c_void_p(back.data_ptr() + j * w * 4), ctypes.c_size_t(nsig * 4),
                        ctypes.c_void_p(dev.data_ptr()), ctypes.c_size_t(w * 4),
                        ctypes.c_size_t(w * 4), ctypes.c_size_t(n))
            if use_kernel:
                nat.call("gsp_stage_cols", *args_in, nat.i32(4), ctypes.c_void_p(st.cuda_stream))
                nat.call("gsp_stage_cols", *args_out, nat.i32(4), ctypes.c_void_p(st.cuda_stream))
            else:
                nat.call("gsp_copy2d_async", *args_in, nat.i32(1), ctypes.c_void_p(st.cuda_stream))
                torch.cuda.synchronize()
                assert torch.equal(dev.cpu(), xh[:, j * w:(j + 1) * w])
                nat.call("gsp_copy2d_async", *args_out, nat.i32(2), ctypes.c_void_p(st.cuda_stream))
        torch.cuda.synchronize()
        assert torch.equal(back, xh)


@pytest.mark.parametrize("stage", ["dma", "kernel"])
@pytest.mark.parametrize("nf", [1, 3])
def test_pinned_host_pipeline_equals_device_path(gsp, monkeypatch, stage, nf):
    """Filter.filter on a pinned host block (column-chunk pipeline, 4 chunks of 16) returns the
    bits of the device-resident path, for one filter (Clenshaw) and for a bank (forward)."""
    import torch
    monkeypatch.setenv("GSPB200_E2E_CHUNK", "16")
    monkeypatch.setenv("GSPB200_STAGE", stage)
    G = gsp.graphs.Sensor(30000, k=8, seed=2, order="morton")
    G.estimate_lmax()
    g = gsp.filters.Heat(G, scale=[10, 20, 40][:nf]) if nf > 1 else gsp.filters.Heat(G, scale=50)
    x = torch.randn(G.N, 64, device="cuda")
    want = g.filter(x, order=20)
    xh = torch.empty(G.N, 64).pin_memory()
    xh.copy_(x)
    for _ in range(2):                       # second call reuses streams / cached blocks
        got = g.filter(xh, order=20)
        assert not got.is_cuda and got.shape == want.shape
        assert torch.equal(got.cuda(), want)
    # and against the oracle
    Lo = G.L.to_scipy().astype(np.float64)
    ref = orc.filter_signal(Lo, G.lmax, orc.heat_kernels(G.lmax, [10, 20, 40][:nf] if nf > 1 else 50),
                            x[:, :4].double().cpu().numpy(), order=20)     # 4 != Nf: signals
    assert relerr_cols(got.numpy()[:, :4].reshape(ref.shape), ref) <= F32_TOL


def test_clenshaw_is_the_default_for_one_filter(gsp, sensor5k):
    """One filter: Filter.filter / cheby_op evaluate by Clenshaw's recurrence unless told
    otherwise; the reference order stays available and both match the oracle."""
    import torch
    from pygsp_b200.filters import approximations as apx
    G, L, _ = sensor5k
    g = gsp.filters.Heat(G, scale=30)
    c = np.atleast_2d(gsp.filters.compute_cheby_coeff(g, m=25))
    x = torch.randn(G.N, 32, device="cuda")
    y = g.filter(x, order=25)
    assert torch.equal(y, apx.cheby_clenshaw_device(G.L, G.lmax, c, x))
    g.clenshaw = False
    y_ref_order = g.filter(x, order=25)
    assert torch.equal(y_ref_order, apx.cheby_op_device(G.L, G.lmax, c, x)[0])
    ref = orc.cheby_op(L, G.lmax, c, x.double().cpu().numpy())
    assert relerr_cols(y.cpu().numpy(), ref) <= F32_TOL
    assert relerr_cols(y_ref_order.cpu().numpy(), ref) <= F32_TOL
    got = apx.cheby_op(G, c[0], x.cpu().numpy())                 # free function, NumPy in / out
    assert relerr_cols(got, ref) <= F32_TOL


@pytest.mark.parametrize("nsig,nscales", [(64, 1), (32, 1), (128, 1), (64, 3), (32, 6), (16, 1)])
def test_tiled_lane_mappings_and_staging_modes_give_the_same_bits(gsp, sensor5k, monkeypatch, nsig, nscales):
    """The tiled step has two lane mappings (one / two float4 packets per lane, GSPB200_TILE_P2)
    and two ways to bring x_old / r (TMA-staged or direct streaming loads, GSPB200_TILE_VDIR).
    Per-row sums run in stored CSR order in all of them: forward recurrence and Clenshaw form
    must agree bit for bit across the four combinations, and with the oracle to 1e-5."""
    import torch
    from pygsp_b200.filters import approximations as apx
    G, L, _ = sensor5k
    rng = np.random.default_rng(77 + nsig + nscales)
    x = torch.from_numpy(rng.standard_normal((G.N, nsig)).astype(np.float32)).cuda()
    c = rng.standard_normal((nscales, 19)) / np.arange(1, 20) ** 2
    got = {}
    for p2 in ("0", "1"):
        for vd in ("0", "1"):
            monkeypatch.setenv("GSPB200_TILE_P2", p2)
            monkeypatch.setenv("GSPB200_TILE_VDIR", vd)
            G.L._plans.clear()
            fwd = apx.cheby_op_device(G.L, G.lmax, c, x)
            cl = apx.cheby_clenshaw_device(G.L, G.lmax, c[:1], x)
            torch.cuda.synchronize()
            got[(p2, vd)] = (fwd.clone(), cl.clone())
    base = got[("0", "0")]
    for key, (fwd, cl) in got.items():
        assert torch.equal(fwd, base[0]), key
        assert torch.equal(cl, base[1]), key
    ref = orc.cheby_op(L, G.lmax, c, x.double().cpu().numpy()).reshape(nscales, G.N, nsig)
    assert relerr_cols(base[0].cpu().numpy().reshape(-1, nsig), ref.reshape(-1, nsig)) <= F32_TOL
    assert relerr_cols(base[1].cpu().numpy(), ref[0]) <= 2 * F32_TOL


def test_spmv_forms_agree(gsp, monkeypatch):
    """The SpMV forms (lane groups walking their row, with 8 or 16 lanes per row / the
    shared-memory x window) against scipy in float64, on a Morton-numbered and on a random graph."""
    import torch
    from scipy import sparse
    rng = np.random.default_rng(9)
    mats = [gsp.graphs.Sensor(30000, k=10, seed=2, order="morton").L,
            gsp.graphs.DeviceCSR.from_scipy(sparse.random(5000, 5000, 0.004, random_state=5, format="csr"),
                                            torch.float32, torch.device("cuda"))]
    for D in mats:
        v = torch.from_numpy(rng.standard_normal(D.shape[1]).astype(np.float32)).cuda()
        out = {}
        for form, lpr in (("subwarp", None), ("subwarp", "16"), ("window", None)):
            monkeypatch.setenv("GSPB200_SPMV", form)
            if lpr:
                monkeypatch.setenv("GSPB200_SPMV_LPR", lpr)
            else:
                monkeypatch.delenv("GSPB200_SPMV_LPR", raising=False)
            out[(form, lpr)] = D.dot(v).clone()
        ref = D.to_scipy().astype(np.float64).dot(v.double().cpu().numpy())
        for key, y in out.items():
            err = np.abs(y.double().cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1e-30)
            assert err <= 2e-6, (key, err)
