"""Golden fixtures for the callers of the filtering path (SURVEY.md 8f rank 3), from the REAL
reference:  PYTHONPATH=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_r2.py

  pyramid.npz  : pygsp.reduction.graph_multiresolution (levels=3, sparsify=False) of a
                 Sensor graph; per level W, lmax, mr['idx'], mr['K_reg']; outputs of
                 reduction.interpolate, pyramid_analysis and (direct) pyramid_synthesis with
                 the Chebyshev method.  The reference's pyramid code only keeps consistent
                 shapes for column-vector signals (N, 1) -- a 1-D signal is silently
                 broadcast to (N, N) at reduction.py:447 -- so signals are given as (N, 1).
  tikhonov.npz : pygsp.learning.regression_tikhonov on a Sensor graph, tau = 3.5 (sparse
                 CG branch, learning.py:326-337) and tau = 0 (learning.py:350-365), plus the
                 exact dense solution of the relaxed problem (the reference's own test oracle,
                 tests/test_learning.py:80-83).
lmax values are computed once by the reference and stored (its ARPACK start vector is unseeded).
"""
import logging
import os

import numpy as np
from scipy import sparse

import pygsp  # noqa: E402
from pygsp import filters, graphs, learning, reduction  # noqa: E402

logging.disable(logging.CRITICAL)
HERE = os.path.dirname(os.path.abspath(__file__))


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    M.sort_indices()
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def pyramid():
    G = graphs.Sensor(256, seed=7)
    G.compute_fourier_basis()
    levels = 3
    Gs = reduction.graph_multiresolution(G, levels, sparsify=False)
    out = {"levels": np.int64(levels)}
    for i, g in enumerate(Gs):
        g.estimate_lmax()
        out.update(csr_parts("W%d" % i, g.W))
        out["lmax%d" % i] = np.float64(g.lmax)
        if i > 0:
            out["idx%d" % i] = np.asarray(g.mr["idx"], dtype=np.int64)
        if "K_reg" in g.mr:
            out["Kreg%d" % i] = np.asarray(sparse.csr_matrix(g.mr["K_reg"]).toarray())
    rng = np.random.default_rng(3)
    f = np.ones((G.N, 1))
    f[: G.N // 2] = -1
    f = f + 0.5 * rng.standard_normal((G.N, 1))
    h = [lambda x: 5.0 / (5 + x)]
    order = 40
    ca, pe = reduction.pyramid_analysis(Gs, f, h_filters=h, order=order)
    rec, ca_rec = reduction.pyramid_synthesis(Gs, ca[levels], pe, order=order)
    out["f"] = f
    out["order"] = np.int64(order)
    for i in range(levels + 1):
        out["ca%d" % i] = np.asarray(ca[i])
    for i in range(levels):
        out["pe%d" % i] = np.asarray(pe[i])
    out["reconstruction"] = np.asarray(rec)
    # interpolate alone (default order 100, Green kernel 1/(eps + x))
    sub = rng.standard_normal((Gs[1].N, 1))
    out["interp_in"] = sub
    out["interp_out"] = reduction.interpolate(Gs[0], sub, Gs[1].mr["idx"])
    sub3 = rng.standard_normal((Gs[1].N, 3))
    cols = [reduction.interpolate(Gs[0], sub3[:, j:j + 1], Gs[1].mr["idx"], order=60) for j in range(3)]
    out["interp3_in"] = sub3
    out["interp3_out"] = np.concatenate(cols, axis=1)          # column by column (see docstring)
    np.savez_compressed(os.path.join(HERE, "pyramid.npz"), **out)


def tikhonov():
    G = graphs.Sensor(100, seed=11)
    G.estimate_lmax()
    filt = filters.Filter(G, lambda x: 1 / (1 + 10 * x))
    rng = np.random.default_rng(1)
    signal = filt.analyze(rng.normal(size=(G.n_vertices, 6)))
    mask = rng.uniform(0, 1, G.n_vertices) > 0.5
    measures = signal.copy()
    measures[~mask] = 18
    tau = 3.5
    out = csr_parts("W", G.W)
    out.update(signal=signal, mask=mask, measures=measures, tau=np.float64(tau))
    out["relaxed_reference_cg"] = learning.regression_tikhonov(G, measures, mask, tau=tau)
    L = G.L.toarray()
    out["relaxed_exact"] = np.linalg.solve(np.diag(1.0 * mask) + tau * L, (mask * measures.T).T)
    nan_measures = signal.copy()
    nan_measures[~mask] = np.nan
    out["constrained_reference"] = learning.regression_tikhonov(G, nan_measures, mask, tau=0)
    out["constrained_1d_reference"] = learning.regression_tikhonov(G, nan_measures[:, 0], mask, tau=0)
    np.savez_compressed(os.path.join(HERE, "tikhonov.npz"), **out)


if __name__ == "__main__":
    print("pygsp", pygsp.__version__)
    pyramid()
    tikhonov()
    for f in ("pyramid.npz", "tikhonov.npz"):
        print(f, os.path.getsize(os.path.join(HERE, f)))
