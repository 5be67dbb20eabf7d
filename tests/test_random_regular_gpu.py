"""RandomRegular on the device (csrc/random_regular.cu): bit for bit against the serial restatement
of oracle/random_regular_oracle.py on every path (bulk rounds, tail, restarts, the last attempt's
switches, the complement, k = 0, 1 and N - 1), independent of the launch shape and of repeated
calls; input errors; the reference's diagnostic; and the spectrum and filtering at N = 10^6."""
import logging

import numpy as np
import pytest

from conftest import relerr_cols
from oracle import pygsp_oracle as orc
from oracle import random_regular_oracle as rro

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5          # the float32 filtering tolerance of tests/test_gpu_parity.py


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


@pytest.fixture
def rg(gsp):
    from pygsp_b200.graphs import random_graphs
    return random_graphs


def _key(seed):
    return int(np.random.default_rng(seed).integers(2 ** 63))


def _same_csr(W, ref):
    S = W.to_scipy()
    assert np.array_equal(S.indptr, ref.indptr)
    assert np.array_equal(S.indices, ref.indices)
    assert np.array_equal(S.data, ref.data)


# name: (N, k, max_iter, seeds); the restart and switch seeds were found with the oracle
CASES = {
    "tail": (64, 6, 10, (0, 7)),
    "tail_dense": (200, 20, 10, (1,)),
    "bulk": (3000, 8, 10, (2, 9)),
    "bulk_large": (20000, 6, 10, (3,)),
    "restart": (16, 6, 10, (1, 25)),
    "switch": (16, 6, 1, (1,)),
    "complement": (16, 9, 10, (5, 6)),
    "complement_bulk": (300, 200, 10, (4,)),
    "k0": (10, 0, 10, (0,)),
    "k1": (10, 1, 10, (0, 1)),
    "k_n_minus_1": (12, 11, 10, (0,)),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_matches_oracle(gsp, rg, monkeypatch, name):
    N, k, max_iter, seeds = CASES[name]
    for seed in seeds:
        ref, attempts, rounds = rro.random_regular_graph(N, k, max_iter, _key(seed))
        if name == "restart":
            assert attempts >= 2
        if name == "switch":
            assert rro.random_regular_graph(N, k, 10, _key(seed))[1] >= 2
        if name.startswith("bulk") or name == "complement_bulk":
            assert rounds >= 1
        for blocks in (0, 1, 0):
            monkeypatch.setattr(rg, "_MAX_BLOCKS", blocks)
            G = gsp.graphs.RandomRegular(N=N, k=k, max_iter=max_iter, seed=seed)
            _same_csr(G.W, ref)
            assert (G._attempts, G._rounds) == (attempts, rounds)
        assert (np.diff(ref.indptr) == k).all() and (ref != ref.T).nnz == 0


def test_attributes_and_dtype(gsp):
    G = gsp.graphs.RandomRegular(seed=42, dtype=np.float64)
    assert (G.N, G.k, G.max_iter, G.seed) == (64, 6, 10, 42)
    assert G._get_extra_repr() == dict(k=6, seed=42)
    assert str(G.W.dtype) == "torch.float64" and not G.is_directed()
    np.testing.assert_equal(np.asarray(G.W.to_scipy().sum(0)).ravel(), 6)   # the reference's test
    np.testing.assert_equal(np.asarray(G.W.to_scipy().sum(1)).ravel(), 6)


def test_errors_before_any_device_call(gsp, rg, monkeypatch):
    called = []
    real = rg.nat.call
    monkeypatch.setattr(rg.nat, "call", lambda name, *a: (called.append(name), real(name, *a)))
    for kw, match in ((dict(N=7, k=3), r"N\*d must be even"), (dict(N=8, k=-2), "non-negative"),
                      (dict(N=6, k=6), "does not exist"), (dict(N=6, k=9), "does not exist"),
                      (dict(N=8, k=2, max_iter=0), "max_iter"),
                      (dict(N=2 ** 27, k=16), "at most 2")):
        with pytest.raises(ValueError, match=match):
            gsp.graphs.RandomRegular(**kw)
    assert called == []


def test_is_regular_logs_the_reference_warning(gsp, caplog):
    with caplog.at_level(logging.WARNING):
        gsp.graphs.RandomRegular(N=30, k=4, seed=1)
    assert not [r for r in caplog.records if "The given matrix" in r.getMessage()]
    with caplog.at_level(logging.WARNING):
        gsp.graphs.RandomRegular.is_regular(gsp.graphs.Path(5))
    msgs = [r.getMessage() for r in caplog.records if "The given matrix" in r.getMessage()]
    assert msgs == ["The given matrix is not d-regular."]
    caplog.clear()
    W = np.array([[0, 2, 1], [0, 1, 0], [1, 0, 0]], dtype=np.float64)
    with caplog.at_level(logging.WARNING):
        gsp.graphs.RandomRegular.is_regular(gsp.graphs.Graph(W))
    msgs = [r.getMessage() for r in caplog.records if "The given matrix" in r.getMessage()]
    assert msgs == ["The given matrix is not symmetric, has parallel edges, is not d-regular, "
                    "has self loop."]


def test_scale_lmax_and_filter(gsp):
    import torch
    from pygsp_b200.graphs.csr import row_ids
    N, k = 10 ** 6, 10
    G = gsp.graphs.RandomRegular(N=N, k=k, seed=0)
    W = G.W
    assert W.nnz == N * k and not G.is_directed() and not G.has_loops()
    assert bool((W.data == 1).all())
    assert (np.diff(W.indptr.cpu().numpy()) == k).all()
    rows = row_ids(W.indptr)
    assert not bool((rows == W.indices.long()).any())
    edge = k + 2 * np.sqrt(k - 1)                      # Friedman: lambda_max(L) -> k + 2 sqrt(k - 1)
    G.estimate_lmax()
    assert abs(G.lmax - 1.01 * edge) <= 0.02 * 1.01 * edge, G.lmax
    # scale 5, not 50: with the spectral gap lambda_2 ~ k - 2 sqrt(k - 1) = 4, exp(-50 lambda_2 /
    # lmax) ~ 4e-6 would leave only the signals' means, a measure of cancellation, not of filtering
    S = W.to_scipy()
    x = np.random.default_rng(0).standard_normal((N, 4)).astype(np.float32)
    y = gsp.filters.Heat(G, 5).filter(x, order=30)
    L = orc.laplacian(S.astype(np.float64))
    ref = orc.filter_signal(L, G.lmax, orc.heat_kernels(G.lmax, 5), x.astype(np.float64),
                            order=30)
    assert relerr_cols(y, ref) <= F32_TOL
    del G, W, rows
    torch.cuda.empty_cache()
