"""Drop-in evidence against the unmodified PyGSP 0.6.1, from stored reference results.

tests/golden/dropin.npz (tests/golden/make_golden_dropin.py) holds (1) the README's Logo
example computed by stock pygsp objects, and (2) a fixed sample of the distinct ``cheby_op``
calls that the reference's own ``pygsp/tests/test_filters.py`` makes, with the SciPy result of
each.  Here (1) is recomputed by this package's Graph / Filter objects, and (2) is replayed
through ``approximations.cheby_op`` on reference-style graph objects (a SciPy ``G.L``), which is
the function ``patch_pygsp()`` binds into a stock pygsp."""
import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


class _ReferenceGraph:
    """What a stock ``pygsp.graphs.Graph`` offers ``cheby_op``: SciPy L, lmax, N."""

    def __init__(self, L, lmax, dtype):
        self.L, self.lmax, self.N = L, lmax, L.shape[0]
        self._gspb200_dtype = dtype


def test_patched_reference_objects(engine, golden):
    import torch
    gsp = engine
    z, logo = golden("dropin"), golden("logo")
    lmax = float(z["obj_lmax"])
    W = csr_from(logo, "W")
    s, rows = z["obj_deltas"], z["obj_rows"]
    block = np.random.default_rng(0).standard_normal((W.shape[0], 7))   # the reference's block
    np.testing.assert_array_equal(block[:, :1], z["obj_block"])          # (its first column is stored)
    want = [z["obj_heat"], z["obj_bank_o40"], z["obj_bank_bank_o25"]]
    shapes = [(W.shape[0],), (W.shape[0], 7, 5), (W.shape[0], 7)]
    for dtype, tol in ((np.float32, 1e-5), (np.float64, 1e-10)):
        G = gsp.graphs.Graph(W, dtype=dtype)
        G._lmax, G._lmax_method = lmax, "lanczos"            # the reference's lmax draw
        bank = gsp.filters.MexicanHat(G, Nf=5)
        heat = gsp.filters.Heat(G, scale=50)
        got = [heat.filter(s), bank.filter(block, order=40),
               bank.filter(bank.filter(block), order=25)]
        for a, b, shape in zip(got, want, shapes):
            a = np.asarray(a, dtype=np.float64)
            assert a.shape == shape
            a = a[rows] if a.ndim == 1 else a[rows, :1]
            assert np.abs(a - b).max() / np.abs(b).max() <= tol
    # the engine's cheby_op on a reference-style graph (what patch_pygsp() routes) returns float64
    c = gsp.filters.compute_cheby_coeff(gsp.filters.Heat(G, scale=50), m=30)
    Lr = csr_from(logo, "logo_Lc")
    y = gsp.filters.approximations.cheby_op(_ReferenceGraph(Lr, lmax, torch.float64), c, s)
    assert y.dtype == np.float64
    assert np.abs(y[rows] - want[0]).max() / np.abs(want[0]).max() <= 1e-10
    # this engine's own Graph against the reference's Graph on the same adjacency
    H = gsp.graphs.Graph(W, dtype=np.float64)
    Lo = H.L.to_scipy()
    np.testing.assert_array_equal(Lo.indptr, Lr.indptr)
    np.testing.assert_array_equal(Lo.indices, Lr.indices)
    np.testing.assert_allclose(Lo.data, Lr.data, rtol=1e-13)
    assert H.n_edges == int(logo["logo_n_edges"])
    assert abs(H._get_upper_bound() - float(logo["logo_bound_c"])) < 1e-9
    H.estimate_lmax()
    assert abs(H.lmax - lmax) / lmax < 2e-4                  # ARPACK's own run-to-run spread is 1e-5


def test_reference_test_suite_on_cuda_engine(engine, golden):
    """Calls of cheby_op made by pygsp/tests/test_filters.py, replayed on the CUDA engine (float64)
    with the reference graph objects' SciPy Laplacians: each result equals the stored SciPy one."""
    import torch
    apx = engine.filters.approximations
    z = golden("dropin")
    n_calls = int(z["suite_calls"])
    assert n_calls >= 24
    graphs = {}
    worst = 0.0
    for i in range(n_calls):
        gi, ci, xi = (int(v) for v in z["suite_%03d_ids" % i])
        if gi not in graphs:
            shape = tuple(int(v) for v in z["suite_L%d_shape" % gi])
            graphs[gi] = sparse.csr_matrix((z["suite_L%d_data" % gi], z["suite_L%d_indices" % gi],
                                            z["suite_L%d_indptr" % gi]), shape=shape)
        G = _ReferenceGraph(graphs[gi], float(z["suite_%03d_lmax" % i]), torch.float64)
        want = z["suite_%03d_y" % i]
        got = apx.cheby_op(G, z["suite_pool_%d" % ci], z["suite_pool_%d" % xi])
        assert got.shape == want.shape and got.dtype == np.float64, i
        err = np.abs(got - want).max() / max(np.abs(want).max(), 1e-300)
        worst = max(worst, err)
        assert err <= 1e-10, (i, err)
    print("replayed %d reference cheby_op calls, worst rel. err %.2e" % (n_calls, worst))
