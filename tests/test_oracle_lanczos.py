"""The Lanczos oracle (oracle/lanczos_oracle.py) against tests/golden/lanczos.npz, the output of
the unmodified PyGSP 0.6.1 -- no GPU needed."""
import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from, load_golden
from oracle import lanczos_oracle as lo

GRAPHS = [str(g) for g in load_golden("lanczos")["graphs"]]
OP_GRAPHS = ("logo", "sensor")


def bank(z, g, name):
    """The fixture's filters, restated: Heat(scale=[5, 20]) and the one-filter step kernel."""
    lmax = float(z[g + "_lmax"])
    if name == "heat":
        return lambda e: np.array([np.exp(-5 * e / lmax), np.exp(-20 * e / lmax)])
    return lambda e: np.array([(e <= 0.3 * lmax) * 1.0])


def relnorm(a, b):
    """Normwise relative difference; an all-zero b (the step kernel at order 1, whose one Ritz
    value lies above the cut) asks for an all-zero a."""
    nb = np.linalg.norm(b)
    return np.linalg.norm(a - b) / nb if nb > 0 else np.linalg.norm(a)


@pytest.mark.parametrize("order", (1, 2, 20))
@pytest.mark.parametrize("g", GRAPHS)
def test_basis_against_reference(golden, g, order):
    z = golden("lanczos")
    V, H, orth = lo.lanczos(csr_from(z, g + "_L"), order, z[g + "_x"])
    ref_V, ref_H = z["%s_V%d" % (g, order)], z["%s_H%d" % (g, order)]
    assert V.shape == ref_V.shape and H.shape == ref_H.shape
    np.testing.assert_allclose(V, ref_V, rtol=1e-8, atol=1e-10)
    np.testing.assert_allclose(H, ref_H, rtol=1e-8, atol=1e-10 * np.abs(ref_H).max())
    np.testing.assert_allclose(orth, z["%s_orth%d" % (g, order)], rtol=1e-6, atol=1e-12)


@pytest.mark.parametrize("order", (1, 10, 30))
@pytest.mark.parametrize("sig", ("s1", "s3"))
@pytest.mark.parametrize("fname", ("heat", "step"))
@pytest.mark.parametrize("g", OP_GRAPHS)
def test_op_against_reference(golden, g, fname, sig, order):
    z = golden("lanczos")
    key = "%s_%s_%s" % (g, fname, sig)
    y = lo.lanczos_op(bank(z, g, fname), csr_from(z, g + "_L"), z["%s_%s" % (g, sig)], order)
    ref = z["%s_o%d" % (key, order)]
    assert y.shape == ref.shape
    assert relnorm(y, ref) <= 1e-9
    if order == 30 and fname == "heat":       # smooth kernel: order 30 is near exact
        assert relnorm(y, z[key + "_exact"]) <= 1e-8


def test_breakdown_is_exact():
    """Ring(8) has 5 distinct eigenvalues, so every Krylov space is invariant after at most 5
    steps.  The reference's early return then hands eig a non-square H and raises; here the
    column freezes and the result is the exact filter output."""
    n = 8
    W = sparse.diags([np.ones(n - 1), np.ones(n - 1)], [1, -1]).tolil()
    W[0, n - 1] = W[n - 1, 0] = 1
    W = W.tocsr()
    L = sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W
    e, U = np.linalg.eigh(L.toarray())
    s = np.random.default_rng(3).standard_normal((n, 2))
    s[:, 1] = 1.0                                # constant: beta_1 = 0 at once
    kern = lambda x: np.array([np.exp(-2 * x), 1 / (1 + x)])   # noqa: E731
    fe = kern(np.maximum(e, 0))
    exact = np.concatenate([U @ (fe[i][:, None] * (U.T @ s)) for i in range(2)])
    y = lo.lanczos_op(kern, L, s, order=20)
    assert np.all(np.isfinite(y))
    np.testing.assert_allclose(y, exact, rtol=0, atol=1e-12)
    _, _, _, m = lo.krylov(L, s, 20)
    assert m[0] <= 5 and m[1] == 1
    # a zero column gives zeros
    y = lo.lanczos_op(kern, L, np.zeros(n), order=5)
    assert y.shape == (2 * n,) and not y.any()


def test_float32_oracle_bound(golden):
    """The float32 bound of tests/test_lanczos_gpu.py comes from this run: the oracle with all
    arithmetic in float32 stays within 1.3e-6 of the fixtures (the engine sums in float64)."""
    z = golden("lanczos")
    worst = 0.0
    for g in OP_GRAPHS:
        for fname in ("heat", "step"):
            for order in (10, 30):
                key = "%s_%s_s3" % (g, fname)
                y = lo.lanczos_op(bank(z, g, fname), csr_from(z, g + "_L"), z[g + "_s3"], order,
                                  dtype=np.float32)
                worst = max(worst, relnorm(y, z["%s_o%d" % (key, order)]))
    assert worst <= 1e-5


def test_lanczos_rejects_a_non_square_matrix():
    """Checked before anything is uploaded, so no device is needed."""
    from pygsp_b200 import filters
    for A in (sparse.random(5, 7, 0.5, random_state=0, format="csr"), np.ones((7, 5))):
        with pytest.raises(ValueError, match="must be square"):
            filters.lanczos(A, 3, np.ones(A.shape[0]))
