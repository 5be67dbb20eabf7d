"""Wide filter banks and the filter designs on the device.  Run on an H100: pytest -m gpu.

  * the stored-basis analysis route (gsp_cheby_op_basis_*) is bit-identical to the same bank in
    groups of at most 16 filters through cheby_op_device, with and without column chunks;
  * the basis route and the wide synthesis (gsp_cheby_synthesis_wide_*) against the float64
    oracle: per column max|y - ref| / max|ref| <= 1e-10 (float64 engine), 1e-5 (float32);
  * every design's Chebyshev and exact analysis against tests/golden/filter_banks.npz (PyGSP
    0.6.1), Gabor and Modulation against oracle/filter_banks_oracle.py on the engine's basis;
  * checks of the reference's test_filters.py, restated.
"""
import logging

import numpy as np
import pytest

from conftest import csr_from, relerr_cols
from oracle import filter_banks_oracle as fbo
from oracle import pygsp_oracle as orc

pytestmark = pytest.mark.gpu

TOL = {np.float32: 1e-5, np.float64: 1e-10}


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


@pytest.fixture(scope="module")
def gold(golden):
    return golden("filter_banks")


def _sensor123(gsp, golden, gold, dtype, basis=False):
    G = gsp.graphs.Graph(csr_from(golden("sensor123"), "W"), dtype=dtype)
    if basis:
        G.compute_fourier_basis()
    G._lmax = float(gold["lmax"])          # the reference's lmax (its e[-1])
    G._lmax_method = "fourier"
    return G


@pytest.fixture(scope="module")
def big(gsp):
    """A graph on which the float32 tiled step applies (several full row tiles)."""
    out = {}
    for dtype in (np.float32, np.float64):
        G = gsp.graphs.Sensor(4096, k=10, seed=0, order="morton", dtype=dtype)
        G.estimate_lmax()
        out[dtype] = G
    return out


def _grouped(apx, L, lmax, c, x):
    import torch
    return torch.cat([apx.cheby_op_device(L, lmax, c[i:i + 16], x)
                      for i in range(0, c.shape[0], 16)])


# ----------------------------------------------------------------- analysis: same bits
@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nf", [17, 33, 100, 1500])
def test_basis_route_bit_identical_to_groups_of_16(gsp, big, dtype, nf):
    import torch
    apx = gsp.filters.approximations
    G = big[dtype]
    L = G.L
    rng = np.random.default_rng(nf)
    c = rng.standard_normal((nf, 31))
    for nsig in (1, 3, 8, 64, 128):
        x = torch.as_tensor(rng.standard_normal((G.N, nsig)), dtype=L.dtype, device=L.device)
        ref = _grouped(apx, L, G.lmax, c, x)
        y = apx.cheby_bank_device(L, G.lmax, c, x)
        assert torch.equal(y, ref), (nf, nsig)
        for cols in (1, 3, 64):
            if cols < nsig:
                assert torch.equal(apx.cheby_bank_device(L, G.lmax, c, x, max_columns=cols), ref)
        del ref, y


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_basis_route_orders(gsp, big, dtype):
    import torch
    apx = gsp.filters.approximations
    G = big[dtype]
    L = G.L
    rng = np.random.default_rng(5)
    x = torch.as_tensor(rng.standard_normal((G.N, 16)), dtype=L.dtype, device=L.device)
    for m in (2, 3, 45, 80):
        c = rng.standard_normal((20, m))
        assert torch.equal(apx.cheby_bank_device(L, G.lmax, c, x), _grouped(apx, L, G.lmax, c, x))
    with pytest.raises(TypeError):
        apx.cheby_bank_device(L, G.lmax, np.ones((20, 1)), x)


# --------------------------------------------------------------- accuracy: float64 oracle
def _heat_bank(G, nf):
    return [lambda x, t=t: np.exp(-t * np.asarray(x) / G.lmax)
            for t in np.linspace(0.5, 30.0, nf)]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_wide_analysis_against_oracle(gsp, golden, gold, dtype):
    G = _sensor123(gsp, golden, gold, dtype)
    L = orc.laplacian(G.W.to_scipy().astype(np.float64))
    kernels = _heat_bank(G, 40)
    g = gsp.filters.Filter(G, kernels)
    s = np.random.default_rng(1).standard_normal((G.N, 5))
    y = g.filter(s, order=30)
    ref = orc.filter_signal(L, G.lmax, kernels, s, order=30)
    assert y.shape == (G.N, 5, 40)
    for j in range(40):
        assert relerr_cols(y[:, :, j], ref[:, :, j]) <= TOL[dtype]
    # the public cheby_op takes the same route for more than 16 coefficient rows
    c = orc.cheby_coeff(kernels, G.lmax, 30)
    r = gsp.filters.cheby_op(G, c, s)
    assert r.shape == (40 * G.N, 5)
    assert relerr_cols(r, orc.cheby_op(L, G.lmax, c, s)) <= TOL[dtype]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nf", [17, 64, 123])
def test_wide_synthesis_against_oracle_and_loop(gsp, golden, gold, dtype, nf):
    G = _sensor123(gsp, golden, gold, dtype)
    assert G.N == 123
    L = orc.laplacian(G.W.to_scipy().astype(np.float64))
    kernels = _heat_bank(G, nf)
    g = gsp.filters.Filter(G, kernels)
    s = np.random.default_rng(nf).standard_normal((G.N, 3, nf))
    y = g.filter(s, order=30)
    ref = orc.filter_signal(L, G.lmax, kernels, s, order=30)
    assert y.shape == (G.N, 3)
    assert relerr_cols(y, ref) <= TOL[dtype]
    g.fused_synthesis = False
    loop = g.filter(s, order=30)
    assert relerr_cols(y, loop) <= 2 * TOL[dtype]
    # the round trip through the device keeps the layout of a CUDA tensor
    import torch
    g.fused_synthesis = True
    yt = g.filter(torch.as_tensor(s, device="cuda"), order=30)
    assert yt.is_cuda and yt.shape == (G.N, 3)
    np.testing.assert_array_equal(yt.cpu().numpy(), y)


# ------------------------------------------------------------------ the reference fixture
DESIGN_NAMES = ["abspline", "expwin", "halfcosine", "held", "itersine", "meyer", "papadakis",
                "rectangular", "regular", "simoncelli", "simpletight", "wave"]


@pytest.fixture(scope="module")
def designs():
    from test_filter_designs_cpu import DESIGNS
    return DESIGNS


@pytest.mark.parametrize("name", DESIGN_NAMES)
def test_design_analysis_matches_reference(gsp, golden, gold, designs, name):
    G = _sensor123(gsp, golden, gold, np.float64, basis=True)
    cls, default, alt = designs[name]
    for key, kwargs in ((name, default), (name + "_alt", alt)):
        f = getattr(gsp.filters, cls)(G, **kwargs)
        cheb = f.filter(gold["signal"], method="chebyshev", order=30).reshape(G.N, -1)
        exact = f.filter(gold["signal"], method="exact").reshape(G.N, -1)
        assert relerr_cols(cheb, gold[key + "_cheby"]) <= 1e-10, key
        np.testing.assert_allclose(exact, gold[key + "_exact"], atol=1e-10, err_msg=key)


def test_gabor_and_modulation(gsp, golden, gold):
    G = _sensor123(gsp, golden, gold, np.float64, basis=True)
    e, U, s = G.e, G.U, gold["signal"]
    rect = gsp.filters.Rectangular(G, None, 0.1)
    delta = gsp.filters.Rectangular(G, 0, 0)
    # Gabor is sign-invariant: the fixture itself
    y = gsp.filters.Gabor(G, rect).filter(s, method="chebyshev", order=10)    # always exact
    assert y.shape == (G.N, G.N)
    np.testing.assert_allclose(y, gold["gabor_rect"], atol=1e-10)
    np.testing.assert_allclose(y, fbo.gabor(e, U, lambda x: rect.evaluate(x)[0], s), atol=1e-12)
    # Modulation, modulation first: the restatement on the engine's basis, and the reference's
    # |Modulation - Gabor| = 0 for the delta kernel
    m1 = gsp.filters.Modulation(G, rect, modulation_first=True)
    np.testing.assert_allclose(m1.filter(s), fbo.modulation_first(e, U, rect.evaluate(e)[0], s),
                               atol=1e-10)
    md = gsp.filters.Modulation(G, delta, modulation_first=True).filter(s)
    np.testing.assert_allclose(np.abs(md), np.abs(gold["gabor_delta"]), atol=1e-10)
    np.testing.assert_allclose(np.abs(md), np.abs(gold["mod_first_delta"]), atol=1e-10)
    np.testing.assert_allclose(np.abs(md), np.abs(gsp.filters.Gabor(G, delta).filter(s)),
                               atol=1e-10)
    # evaluate: the table at the eigenvalues, NaN elsewhere
    r = m1.evaluate(np.array([e[3], 0.5 * (e[3] + e[4])]))
    np.testing.assert_allclose(r[:, 0], fbo.modulation_table(e, U, rect.evaluate(e)[0])[3],
                               atol=1e-12)
    assert np.all(np.isnan(r[:, 1]))
    # the windowed graph Fourier transform: windows sqrt(N) g(L) I by the order-30 expansion
    L = orc.laplacian(G.W.to_scipy().astype(np.float64))
    windows = orc.filter_signal(L, G.lmax, [lambda x: rect.evaluate(x)[0]], np.identity(G.N))
    windows *= np.sqrt(G.N)
    m2 = gsp.filters.Modulation(G, rect)
    y2 = m2.filter(s)
    assert y2.shape == (G.N, G.N)
    np.testing.assert_allclose(y2, fbo.windowed_gft(U, windows, s), atol=1e-10)
    with pytest.raises(ValueError):
        m2.filter(np.ones((G.N, 2)))
    # a kernel of several filters, or one built on another graph, is refused
    other = gsp.graphs.Graph(csr_from(golden("sensor123"), "W"), dtype=np.float64)
    for bank in (gsp.filters.Gabor, gsp.filters.Modulation):
        with pytest.raises(ValueError):
            bank(G, gsp.filters.Regular(G))
        with pytest.raises(ValueError):
            bank(other, rect)


# ------------------------------------------------------------- checks of test_filters.py
def test_frame_methods_on_a_graph(gsp, golden, gold, caplog):
    G = _sensor123(gsp, golden, gold, np.float64, basis=True)
    assert gsp.filters.Rectangular(G).estimate_frame_bounds() == (0, 1)
    assert gsp.filters.Filter(G, lambda x: np.full_like(x, 2)).estimate_frame_bounds() == (4, 4)
    mh = gsp.filters.MexicanHat(G)
    mh += mh.complement(2.5)
    np.testing.assert_allclose(mh.estimate_frame_bounds(), (2.5, 2.5))
    g = gsp.filters.Heat(G, scale=[2, 3, 4])
    h = g.inverse()
    Ag, Bg = g.estimate_frame_bounds()
    Ah, Bh = h.estimate_frame_bounds()
    np.testing.assert_allclose([Ag * Bh, Bg * Ah], [1, 1], rtol=1e-10)
    gL = g.compute_frame(method="exact")
    hL = h.compute_frame(method="exact")
    np.testing.assert_allclose(hL.T @ gL, np.identity(G.N), atol=1e-10)
    np.testing.assert_allclose(np.linalg.inv(gL.T @ gL) @ gL.T, hL.T, atol=1e-10)
    np.testing.assert_allclose(g.toarray(), g.compute_frame(), atol=0)
    s = gold["signal"]
    z = h.filter(g.filter(s, method="exact"), method="exact")
    np.testing.assert_allclose(z, s, atol=1e-10)
    with caplog.at_level(logging.WARNING):
        gsp.filters.Expwin(G).inverse()
    assert any("not invertible" in r.getMessage() for r in caplog.records)
