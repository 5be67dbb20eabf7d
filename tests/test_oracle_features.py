"""The features oracle (oracle/features_oracle.py) against tests/golden/features.npz, the output
of the unmodified PyGSP 0.6.1, and the host half of the engine's moment route -- no GPU needed."""
import numpy as np
from numpy.polynomial import chebyshev as npcheb
from scipy import sparse

from conftest import csr_from, relerr_cols
from oracle import features_oracle as fo

TOL = 1e-12


class FakeGraph:
    def __init__(self, lmax, N):
        self.lmax, self.N = lmax, N


def sensor(z):
    """(L, lmax) of the fixture's Sensor(300), combinatorial Laplacian of its W."""
    W = csr_from(z, "sensor_W")
    L = sparse.csgraph.laplacian(W).tocsr()
    return L, float(z["sensor_lmax"])


def kernels(name, lmax, N):
    from pygsp_b200 import filters
    G = FakeGraph(lmax, N)
    f = filters.Heat(G, scale=10) if name == "heat" else filters.MexicanHat(G, Nf=3)
    return f._kernels


def atom(lmax):
    return lambda x: 1.0 / (1.0 + (10.0 * x / lmax) ** 2)


def test_spectrogram_frame_route(golden):
    z = golden("features")
    L, lmax = sensor(z)
    assert relerr_cols(fo.spectrogram_frame(L, lmax), z["spectr_default"]) <= TOL
    assert relerr_cols(fo.spectrogram_frame(L, lmax, atom(lmax), M=20), z["spectr_atom"]) <= TOL


def test_norm_tig_frame_route(golden):
    z = golden("features")
    L, lmax = sensor(z)
    assert relerr_cols(fo.norm_tig_frame(L, lmax, kernels("heat", lmax, 300)),
                       z["norm_heat"]) <= TOL
    mh = fo.norm_tig_frame(L, lmax, kernels("mh", lmax, 300))
    for ref in z["norm_mh"]:                 # Nf copies of the whole (N Nf,) vector
        assert relerr_cols(mh, ref) <= TOL


def test_moment_route_matches_the_reference(golden):
    """Every vertex of the Sensor(300) by moments against the reference's frame, per column."""
    z = golden("features")
    L, lmax = sensor(z)
    cols = np.arange(300)
    sq = fo.square_norms_moments(L, lmax, fo.spectrogram_kernels(lmax), cols)
    assert relerr_cols(sq, z["spectr_default"]) <= TOL
    sq = fo.square_norms_moments(L, lmax, fo.spectrogram_kernels(lmax, atom(lmax), 20), cols)
    assert relerr_cols(sq, z["spectr_atom"]) <= TOL
    sq = fo.square_norms_moments(L, lmax, kernels("mh", lmax, 300), cols)
    assert relerr_cols(np.sqrt(sq).T.reshape(-1), z["norm_mh"][0]) <= TOL


def test_cheby_square_coeff():
    """The engine's host series of p^2 against numpy's Chebyshev product, and p^2 itself."""
    from pygsp_b200.filters.approximations import cheby_square_coeff
    rng = np.random.default_rng(0)
    for m in (1, 2, 7, 30, 50):
        c = rng.standard_normal(m + 1)
        d = cheby_square_coeff(c)
        a = c.copy()
        a[0] *= 0.5
        e = npcheb.chebmul(a, a)
        assert d.shape == (2 * m + 1,)
        np.testing.assert_allclose(d[1:], e[1:], rtol=1e-13, atol=1e-13 * np.abs(e).max())
        assert abs(d[0] / 2 - e[0]) <= 1e-13 * np.abs(e).max()
        x = np.linspace(-1, 1, 17)
        np.testing.assert_allclose(npcheb.chebval(x, e), npcheb.chebval(x, a) ** 2,
                                   rtol=1e-12, atol=1e-12)
    C = rng.standard_normal((4, 11))
    D = cheby_square_coeff(C)
    assert D.shape == (4, 21)
    np.testing.assert_array_equal(D[2], cheby_square_coeff(C[2]))


def test_avg_adj_deg(golden):
    z = golden("features")
    for g in ("sensor", "directed", "isolated"):
        ref = z["adj_" + g]
        got = fo.avg_adj_deg(csr_from(z, "adj_%s_W" % g))
        assert got.shape == ref.shape == (ref.shape[0], 1)
        np.testing.assert_array_equal(got, ref)
    # the path 0 - 1 - 2 (a distinct-endpoint count, not a walk count)
    W = sparse.csr_matrix(np.array([[0, 1, 0], [1, 0, 1], [0, 1, 0]], dtype=float))
    np.testing.assert_array_equal(fo.avg_adj_deg(W).ravel(), [1, 1 / 3, 1])
