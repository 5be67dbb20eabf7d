"""Wide filter banks and the filter designs on the device.  Run on an H100: pytest -m gpu.

  * the stored-basis analysis route (gsp_cheby_op_basis_*) is bit-identical to the same bank in
    groups of at most 16 filters through cheby_op_device, with and without column chunks, at
    orders that run the combine at 128, 64 and 32 threads and in several order chunks;
  * the wide synthesis (gsp_cheby_synthesis_wide_*) gives the bits of the row-group kernel on the
    tiled step at every tiled width and under the tiled launch variants; its per-order sources,
    read back from the work buffer, and its last step are held to proven bounds
    (oracle/step_oracle.py);
  * the 16/17 filter route boundary, NumPy / CUDA / page-locked inputs and the fused step with
    more than 16 scales (cheby_axpy_scales) give the bits of the basis route or match the oracle;
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
from oracle import step_oracle as so

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


# the combine stages 16 B per order and thread when vectorised (float32 with nsig % 4 == 0,
# float64 with even nsig): 128 threads up to m = 113, 64 up to 227, 32 up to 454, then order
# chunks of 454.  Unvectorised float32 (4 B) halves at 454 and 908 and chunks past 1816; float64
# (8 B) halves at 227 and 454 and chunks past 908.
COMBINE_ORDERS = (113, 114, 227, 228, 454, 455, 1000)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_basis_route_orders(gsp, big, dtype):
    """Same bits as groups of 16 at every thread count of the combine and in order chunks, with
    and without the vectorised path and column chunks; no order limit."""
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
    # an upper bound of the spectrum keeps T_k x bounded at order 999
    lmax = 1.01 * float(abs(L.to_scipy().astype(np.float64)).sum(axis=1).max())
    for nsig in (3, 4, 16):
        xs = x[:, :nsig].contiguous()
        for m in COMBINE_ORDERS:
            c = rng.standard_normal((20, m)) / np.arange(1, m + 1)
            ref = _grouped(apx, L, lmax, c, xs)
            assert torch.isfinite(ref).all()
            assert torch.equal(apx.cheby_bank_device(L, lmax, c, xs), ref), (nsig, m)
            if m == 455 and nsig == 16:
                for cols in (4, 6):
                    y = apx.cheby_bank_device(L, lmax, c, xs, max_columns=cols)
                    assert torch.equal(y, ref), (cols, m)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_high_order_bank_does_not_depend_on_the_width(gsp, big, dtype):
    """Order 500 on a 20-filter bank: 4 columns (vectorised combine, in two order chunks) give
    the bits of the same 3 columns (one chunk at 128 or 64 threads) and of groups of 16."""
    import torch
    G = big[dtype]
    g = gsp.filters.Filter(G, _heat_bank(G, 20))
    s = np.random.default_rng(8).standard_normal((G.N, 4))
    y4 = g.filter(s, order=500)
    y3 = g.filter(s[:, :3], order=500)
    assert y4.shape == (G.N, 4, 20) and y3.shape == (G.N, 3, 20)
    assert np.isfinite(y4).all()
    np.testing.assert_array_equal(y4[:, :3], y3)
    apx = gsp.filters.approximations
    c = apx.compute_cheby_coeff(g, m=500)
    x = torch.as_tensor(s, dtype=G.L.dtype, device=G.L.device)
    np.testing.assert_array_equal(
        _grouped(apx, G.L, G.lmax, np.asarray(c), x).permute(1, 2, 0).cpu().numpy(), y4)


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


# ------------------------------------------- wide synthesis on the tiled step and its pieces
WIDTHS = (8, 16, 32, 64, 128)                    # the tiled step's widths
SYN_ORDERS = (1, 2, 3, 7, 8, 15, 16, 30, 31, 32, 33, 64)   # m = 2 .. 65: KP 8/16/32, 1-3 passes
GRAPHS = ["morton k-NN", "rows past the last tile", "renumbered", "one-way edges"]


@pytest.fixture(scope="module")
def tiled_graphs(gsp):
    """The float32 Laplacians of the paired-launch tests, on the device, with an upper bound of
    their spectra (name -> (scipy L, lmax, DeviceCSR))."""
    import torch
    from test_clenshaw_pairs_gpu import _graphs
    out = {}
    for name, Lh in _graphs().items():
        lmax = 1.01 * float(abs(Lh.astype(np.float64)).sum(axis=1).max())
        out[name] = (Lh, lmax, gsp.graphs.DeviceCSR.from_scipy(Lh, torch.float32,
                                                               torch.device("cuda")))
    return out


def _rowgroup_csr(gsp, monkeypatch, Lh, dtype=np.float32):
    """A DeviceCSR planned under GSPB200_KERNEL=rowgroup: every step runs the row-group kernel."""
    import torch
    tdt = torch.float32 if dtype == np.float32 else torch.float64
    dev = gsp.graphs.DeviceCSR.from_scipy(Lh.astype(dtype), tdt, torch.device("cuda"))
    with monkeypatch.context() as m:
        m.setenv("GSPB200_KERNEL", "rowgroup")
        for nsig in WIDTHS:
            assert dev.tile_plan(nsig, 1) is None
    return dev


def _sources(rng, nf, n, nsig, dtype=np.float32):
    import torch
    return torch.from_numpy(np.stack([so.scaled_signals(rng, n, nsig, dtype)
                                      for _ in range(nf)])).cuda()


def _coeffs(rng, nf, m):
    return rng.standard_normal((nf, m)) / np.arange(1, m + 1)


def _wide_call(gsp, L, lmax, c, src):
    """gsp_cheby_synthesis_wide_* with a caller-owned work buffer (m + 2, N, nsig), filled with
    NaN first: returns (out, work) after the call."""
    import torch
    nat = gsp._native
    c = np.ascontiguousarray(np.atleast_2d(c), dtype=np.float64)
    nsrc, m = c.shape
    _, n, nsig = src.shape
    out = torch.full((n, nsig), float("nan"), dtype=L.dtype, device=L.device)
    work = torch.full((m + 2, n, nsig), float("nan"), dtype=L.dtype, device=L.device)
    with torch.cuda.device(L.device):
        nat.call("gsp_cheby_synthesis_wide_" + nat.suffix(L.dtype), nat.i64(n), nat.i64(L.nnz),
                 L.indptr, L.indices, L.data, nat.f64(lmax), torch.as_tensor(c, device=L.device),
                 nat.i32(nsrc), nat.i32(m), src, nat.i64(nsig), out, work, L.tile_plan(nsig, 1),
                 nat.stream_ptr(L.device))
    torch.cuda.synchronize()
    return out, work


@pytest.mark.parametrize("name", GRAPHS)
def test_wide_synthesis_tiled_gives_the_rowgroup_bits(gsp, tiled_graphs, monkeypatch, name):
    """The recurrence of the wide synthesis on the tiled step (a source block that moves every
    step, rows past the last full tile) against the row-group kernel, bit for bit, at every
    tiled width, for m = 2 .. 65; then under every tiled launch variant."""
    import torch
    from test_tiled_step_gpu import VARIANTS
    apx = gsp.filters.approximations
    lib = gsp._native.lib()
    Lh, lmax, dev = tiled_graphs[name]
    n = Lh.shape[0]
    rowgroup = _rowgroup_csr(gsp, monkeypatch, Lh)
    rng = np.random.default_rng(17)
    refs = {}
    for nsig in WIDTHS:
        assert dev.tile_plan(nsig, 1) is not None, nsig
        for nf in (17, 33):
            src = _sources(rng, nf, n, nsig)
            for order in SYN_ORDERS:
                c = _coeffs(rng, nf, order + 1)
                before = lib.gsp_launch_count()
                y = apx.cheby_synthesis_wide_device(dev, lmax, c, src)
                mid = lib.gsp_launch_count()
                ref = apx.cheby_synthesis_wide_device(rowgroup, lmax, c, src)
                torch.cuda.synchronize()
                end = lib.gsp_launch_count()
                assert torch.equal(y, ref), (nsig, nf, order, int((y != ref).sum()))
                if name == "rows past the last tile":
                    # each tiled step is a tiled launch plus a row-group launch for the tail
                    assert mid - before > end - mid, (nsig, order)
                if nf == 17 and nsig in (8, 64, 128) and order in (2, 33):
                    refs[nsig, order] = (c, src, ref)
    variants = [v for v in VARIANTS if "GSPB200_FORCE_HALO" not in v]
    try:
        for env in variants:
            with monkeypatch.context() as m:
                for k, v in env.items():
                    m.setenv(k, v)
                dev._plans.clear()
                for (nsig, order), (c, src, ref) in refs.items():
                    y = apx.cheby_synthesis_wide_device(dev, lmax, c, src)
                    assert torch.equal(y, ref), (env, nsig, order)
    finally:
        dev._plans.clear()


def _mix_check(gsp, L, lmax, dtype, src, m, nsrc, rng):
    c = _coeffs(rng, nsrc, m)
    _, work = _wide_call(gsp, L, lmax, c, src)
    u, bound = so.mix_reference(src.cpu().numpy(), c, dtype)
    got = work[:m].cpu().numpy()
    bad = so.violations(got, u, bound)
    assert not bad.any(), (m, nsrc, np.argwhere(bad)[:3].tolist())


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_wide_synthesis_mix_within_bound(gsp, monkeypatch, dtype):
    """The per-order sources u_k = sum_f c'_fk s_f (c'_f0 = c_f0 / 2), read back from work[:m]
    after the call, within gamma_nsrc sum_f |c'_fk s_f| of a wide-type reference: one, two and
    four order passes of KP = 8, 16 and 32, across the 32-row staging of the coefficients, on a
    block of 300 x 3 elements (not a multiple of the 256-thread CTA) and of 512 x 8."""
    Lh = orc.laplacian(so.sensor_adjacency(300, k=6, seed=2)).astype(dtype)
    lmax = 1.01 * float(abs(Lh.astype(np.float64)).sum(axis=1).max())
    L = _rowgroup_csr(gsp, monkeypatch, Lh, dtype)
    rng = np.random.default_rng(23)
    for nsrc in (17, 31, 32, 33, 64, 65):
        src = _sources(rng, nsrc, 300, 3, dtype)
        for m in (2, 8, 9, 16, 17, 32, 33, 64, 65, 100):
            _mix_check(gsp, L, lmax, dtype, src, m, nsrc, rng)
    Lh = orc.laplacian(so.sensor_adjacency(512, k=6, seed=3)).astype(dtype)
    L = gsp.graphs.DeviceCSR.from_scipy(Lh, L.dtype, L.device)
    lmax = 1.01 * float(abs(Lh.astype(np.float64)).sum(axis=1).max())
    for nsrc in (32, 33):
        src = _sources(rng, nsrc, 512, 8, dtype)
        for m in (33, 65):
            _mix_check(gsp, L, lmax, dtype, src, m, nsrc, rng)


@pytest.mark.parametrize("dtype,name", [(np.float32, g) for g in GRAPHS]
                         + [(np.float64, "rows past the last tile")])
def test_wide_synthesis_last_step_within_bound(gsp, tiled_graphs, monkeypatch, dtype, name):
    """out = (2/lmax) L b_1 - b_1 - b_2 + u_0 from the b_1, b_2 and u_0 the call left in its
    work buffer, against the step reference with one source term (float32 on the tiled kernel
    at every width, float64 on the row-group kernel): K = 1 (b_1 = u_1, no b_2), K = 2
    (b_2 = u_2) and both parities of K >= 3."""
    Lh, lmax, dev = tiled_graphs[name]
    if dtype == np.float64:
        dev = _rowgroup_csr(gsp, monkeypatch, Lh, dtype)
    Le = Lh.astype(dtype)
    n = Lh.shape[0]
    rng = np.random.default_rng(29)
    for nsig in WIDTHS:
        src = _sources(rng, 17, n, nsig, dtype)
        for K in (1, 2, 3, 8, 33):
            m = K + 1
            c = _coeffs(rng, 17, m)
            out, work = _wide_call(gsp, dev, lmax, c, src)
            w = work.cpu().numpy()
            if K == 1:
                b1, b2, gamma = w[1], w[1], 0.0
            elif K == 2:
                b1, b2, gamma = w[m], w[2], -1.0
            else:
                b1, b2, gamma = w[m + ((K - 2) & 1)], w[m + ((K - 3) & 1)], -1.0
            x, _, bx, _ = so.step_reference(Le, b1, b2, None, 2.0 / lmax, -1.0, gamma, [], [],
                                            False, dtype=dtype, sources=w[:1], cs=[1.0])
            bad = so.violations(out.cpu().numpy(), x, bx)
            assert not bad.any(), (nsig, K, np.argwhere(bad)[:3].tolist())


def _heat(lmax, nf):
    return [lambda x, t=t: np.exp(-t * np.asarray(x) / lmax) for t in np.linspace(0.5, 30.0, nf)]


@pytest.mark.parametrize("name", GRAPHS)
def test_wide_synthesis_whole_calls_against_oracle(gsp, tiled_graphs, monkeypatch, name):
    """Heat banks of 17 and 33 filters up to order 64 on the graphs of the tiled tests: the
    float32 engine (tiled step) within 1e-5 and the float64 engine within 1e-10 of
    orc.filter_signal, per column."""
    import torch
    apx = gsp.filters.approximations
    Lh, lmax, dev = tiled_graphs[name]
    dev64 = gsp.graphs.DeviceCSR.from_scipy(Lh.astype(np.float64), torch.float64,
                                            torch.device("cuda"))
    L64 = Lh.astype(np.float64)
    n = Lh.shape[0]
    rng = np.random.default_rng(31)
    for nf, order in ((17, 2), (17, 33), (33, 64)):
        kernels = _heat(lmax, nf)
        s = np.stack([so.scaled_signals(rng, n, 8) for _ in range(nf)], axis=2)    # (n, 8, nf)
        ref = orc.filter_signal(L64, lmax, kernels, s.astype(np.float64), order=order)
        c = orc.cheby_coeff(kernels, lmax, order)
        for L, tol in ((dev, TOL[np.float32]), (dev64, TOL[np.float64])):
            src = torch.as_tensor(np.ascontiguousarray(s.transpose(2, 0, 1)), dtype=L.dtype,
                                  device=L.device)
            y = apx.cheby_synthesis_wide_device(L, lmax, c, src).cpu().numpy()
            assert relerr_cols(y, ref) <= tol, (nf, order, L.dtype, relerr_cols(y, ref))


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_filter_route_boundary_16_17(gsp, big, dtype):
    """Filter.filter with 16 filters (fused step, multi-source Clenshaw) and 17 (basis route,
    wide synthesis): analysis and synthesis both match the float64 oracle."""
    G = big[dtype]
    L = orc.laplacian(G.W.to_scipy().astype(np.float64))
    rng = np.random.default_rng(37)
    for nf in (16, 17):
        kernels = _heat_bank(G, nf)
        g = gsp.filters.Filter(G, kernels)
        s = rng.standard_normal((G.N, 4))
        y = g.filter(s, order=30)
        ref = orc.filter_signal(L, G.lmax, kernels, s, order=30)
        assert y.shape == (G.N, 4, nf)
        for j in range(nf):
            assert relerr_cols(y[:, :, j], ref[:, :, j]) <= TOL[dtype], (nf, j)
        s3 = rng.standard_normal((G.N, 4, nf))
        y3 = g.filter(s3, order=30)
        assert y3.shape == (G.N, 4)
        assert relerr_cols(y3, orc.filter_signal(L, G.lmax, kernels, s3, order=30)) <= TOL[dtype]


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nf", [17, 40])
def test_analysis_same_bits_for_every_input_kind(gsp, big, dtype, nf):
    """A NumPy array and a CUDA tensor (basis route) and a page-locked host tensor (the pinned
    pipeline: the fused step plus cheby_axpy_scales) give the same bits."""
    import torch
    G = big[dtype]
    g = gsp.filters.Filter(G, _heat_bank(G, nf))
    s = np.random.default_rng(nf).standard_normal((G.N, 8)).astype(dtype)
    y = g.filter(s, order=30)
    yt = g.filter(torch.as_tensor(s, device="cuda"), order=30)
    pinned = torch.from_numpy(s).pin_memory()
    yp = g.filter(pinned, order=30)
    assert yt.is_cuda and not yp.is_cuda
    assert y.shape == tuple(yt.shape) == tuple(yp.shape) == (G.N, 8, nf)
    np.testing.assert_array_equal(yt.cpu().numpy(), y)
    np.testing.assert_array_equal(yp.numpy(), y)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("nscales", [17, 33])
def test_cheby_op_device_wide_scales(gsp, big, dtype, nscales):
    """cheby_op_device with more than 16 scales (the fused step on the first 16, cheby_axpy_scales
    on the rest) gives the bits of the basis route and matches the oracle."""
    import torch
    apx = gsp.filters.approximations
    G = big[dtype]
    L = G.L
    rng = np.random.default_rng(41 + nscales)
    c = rng.standard_normal((nscales, 21)) / np.arange(1, 22) ** 2
    for nsig in (3, 16):
        x = rng.standard_normal((G.N, nsig))
        xt = torch.as_tensor(x, dtype=L.dtype, device=L.device)
        y = apx.cheby_op_device(L, G.lmax, c, xt)
        assert torch.equal(y, apx.cheby_bank_device(L, G.lmax, c, xt)), nsig
        ref = orc.cheby_op(L.to_scipy().astype(np.float64), G.lmax, c, xt.double().cpu().numpy())
        assert relerr_cols(y.reshape(nscales * G.N, nsig).cpu().numpy(), ref) <= TOL[dtype]


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
