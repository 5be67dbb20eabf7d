"""Generate the golden fixtures under tests/golden/ from the REAL reference.

Run once on any machine with a PyGSP 0.6.1 source tree (no GPU needed):

    PYTHONPATH=<PyGSP 0.6.1 source tree> python tests/golden/make_golden.py

Every array saved here is an output of unmodified PyGSP 0.6.1 code
(`pygsp.graphs.Graph`, `pygsp.filters.*`, `pygsp.filters.approximations`).
lmax is always computed ONCE by the reference and stored, because the
reference's `estimate_lmax` is not reproducible run to run (unseeded ARPACK
start vector), and every consumer (oracle, CUDA engine) is given that value.
"""

import logging
import os

import numpy as np
from scipy import sparse

import pygsp  # noqa: E402
from pygsp import filters, graphs  # noqa: E402
from pygsp.filters import approximations  # noqa: E402

logging.disable(logging.CRITICAL)
HERE = os.path.dirname(os.path.abspath(__file__))


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def lap_parts(prefix, W, **kw):
    out = {}
    for lap in ("combinatorial", "normalized"):
        G = graphs.Graph(W, lap_type=lap, **kw)
        out.update(csr_parts(prefix + "_L" + lap[0], G.L))
        out[prefix + "_bound_" + lap[0]] = np.float64(G._get_upper_bound())
    out[prefix + "_dw"] = np.asarray(G.dw, dtype=np.float64)
    out[prefix + "_d"] = np.asarray(G.d, dtype=np.float64)
    out[prefix + "_directed"] = np.bool_(G.is_directed())
    out[prefix + "_n_edges"] = np.int64(G.n_edges)
    return out


def logo():
    """BASELINE config 1: README.rst:68-89."""
    G = graphs.Logo()
    out = csr_parts("W", G.W)
    out.update(lap_parts("logo", G.W))
    G.compute_fourier_basis()
    out["lmax_exact"] = np.float64(G.lmax)
    G2 = graphs.Logo()
    G2.estimate_lmax()
    out["lmax_lanczos"] = np.float64(G2.lmax)        # one draw of the reference
    g = filters.Heat(G2, scale=50)
    s = np.zeros(G2.N)
    s[[20, 30, 1090]] = 1
    out["heat50_coeff"] = approximations.compute_cheby_coeff(g, m=30)
    out["readme_signal"] = s
    out["readme_filtered"] = g.filter(s)             # chebyshev, order 30
    # cheby_rect (approximations.py:117-163) on the same graph / lmax
    sig = np.random.default_rng(7).standard_normal((G2.N, 3))
    out["rect_signal"] = sig
    out["rect_bounds"] = np.array([2.0, 6.0])
    out["rect_filtered"] = approximations.cheby_rect(G2, [2.0, 6.0], sig, order=25)
    np.savez_compressed(os.path.join(HERE, "logo.npz"), **out)


def sensor123():
    """Fixtures of pygsp/tests/test_filters.py:12-29 plus shape truth table."""
    G = graphs.Sensor(123, seed=42)
    G.compute_fourier_basis()
    rng = np.random.default_rng(42)
    signal = rng.uniform(size=G.N)
    out = csr_parts("W", G.W)
    out.update(lap_parts("s", G.W))
    out["lmax"] = np.float64(G.lmax)
    out["signal"] = signal
    # test_approximations (test_filters.py:403-417): Heat() order 30 vs exact
    g = filters.Heat(G)
    out["heat10_cheb"] = g.filter(signal, method="chebyshev")
    out["heat10_exact"] = g.filter(signal, method="exact")
    out["heat10_coeff"] = approximations.compute_cheby_coeff(g, m=30)
    # test_frame (:157-168): Heat(scale=[8, 9])
    g = filters.Heat(G, scale=[8, 9])
    out["heat89_coeff"] = np.array(approximations.compute_cheby_coeff(g, m=30))
    out["heat89_frame"] = g.compute_frame(method="chebyshev", order=30)
    # MexicanHat bank, analysis + synthesis on a signal block
    g = filters.MexicanHat(G, Nf=5)
    out["mh5_coeff"] = np.array(approximations.compute_cheby_coeff(g, m=40))
    block = rng.standard_normal((G.N, 3))
    out["mh5_block"] = block
    out["mh5_analysis"] = g.filter(block, order=40)            # (N, 3, 5)
    out["mh5_synthesis"] = g.filter(out["mh5_analysis"], order=40)   # (N, 3)
    # raw cheby_op with a coefficient matrix
    out["mh5_cheby_op"] = approximations.cheby_op(G, out["mh5_coeff"], block)
    # shape truth table of Filter.filter (SURVEY.md 3.5)
    g1 = filters.Heat(G, 10)
    shapes = [(G.N,), (G.N, 1), (G.N, 3), (G.N, 7), (G.N, 5), (G.N, 3, 1),
              (G.N, 1, 5), (G.N, 3, 5), (G.N, 5, 1)]
    for j, shp in enumerate(shapes):
        x = np.random.default_rng(100 + j).standard_normal(shp)
        out["tt%d_in" % j] = x
        out["tt%d_mh5" % j] = g.filter(x, order=20)
        if not (len(shp) > 1 and shp[-1] == 5):
            out["tt%d_heat" % j] = g1.filter(x, order=20)
    # localize (filter.py:350-391)
    out["localize_7"] = g1.localize(7, order=25)
    np.savez_compressed(os.path.join(HERE, "sensor123.npz"), **out)


def doctest_027649():
    """filter.py:232-256 -- Heat -> MexicanHat analyze -> synthesize == 0.27649."""
    G = graphs.Sensor(30, seed=42)
    G.compute_fourier_basis()
    s1 = np.zeros(G.N)
    s1[13] = 1
    s1 = filters.Heat(G, 3).filter(s1)
    g = filters.MexicanHat(G, Nf=4)
    s2 = g.analyze(s1)
    s3 = g.synthesize(s2)
    out = csr_parts("W", G.W)
    out.update(lmax=np.float64(G.lmax), s1=s1, s2=s2, s3=s3,
               norm=np.float64(np.linalg.norm(s1 - s3)))
    # filter.py:213-219 -- Ring(60), Heat taus [1, 10, 100], (60, 10) -> (60, 10, 3)
    R = graphs.Ring(N=60)
    R.estimate_lmax()
    s = np.random.default_rng(42).uniform(size=(R.N, 10))
    out.update(csr_parts("ringW", R.W))
    out.update(ring_lmax=np.float64(R.lmax), ring_signal=s,
               ring_filtered=filters.Heat(R, [1, 10, 100]).filter(s))
    np.savez_compressed(os.path.join(HERE, "doctest.npz"), **out)


def laplacian_kats():
    """pygsp/tests/test_graphs.py:195-254 + graph.py doctests + edge cases."""
    out = {}
    cases = {
        "undir4": [[0, 3, 0, 1], [3, 0, 1, 0], [0, 1, 0, 3], [1, 0, 3, 0]],
        "dir4": [[0, 6, 0, 1], [0, 0, 0, 0], [0, 2, 0, 3], [1, 0, 3, 0]],
        "doc3": [[0., 2., 0.], [2., 0., 5.], [0., 5., 0.]],
        "isolated": [[0, 1, 0, 0], [1, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, 0]],
        "loops": [[2, 1, 0], [1, 0, 3], [0, 3, 1.5]],
        "onlyloop": [[4., 0, 0], [0, 0, 1], [0, 1, 0]],
        "negative": [[0, -1, 2], [-1, 0, 0.5], [2, 0.5, 0]],
        "dircancel": [[0, 1., 0], [-1., 0, 2], [0, 0, 0]],
        "empty": np.zeros((5, 5)),
        "full10": np.full((10, 10), 2),
        "bip_reg": [[0, 0, 1, 1], [0, 0, 1, 1], [1, 1, 0, 0], [1, 1, 0, 0]],
        "bip": [[0, 0, 1, 1], [0, 0, 1, 0], [1, 1, 0, 0], [1, 0, 0, 0]],
    }
    rng = np.random.default_rng(3)
    A = sparse.random(60, 60, 0.08, random_state=3, format="csr")
    cases["rand_dir"] = A.toarray()
    B = sparse.random(80, 80, 0.06, random_state=4, format="csr")
    B = B + B.T
    B.setdiag(rng.uniform(size=80) * (rng.uniform(size=80) < 0.2))
    cases["rand_undir_loops"] = B.toarray()
    out["names"] = np.array(sorted(cases))
    for name, A in cases.items():
        A = np.asarray(A, dtype=np.float64)
        out[name + "_A"] = A
        out.update(lap_parts(name, A))
    np.savez_compressed(os.path.join(HERE, "laplacian_kat.npz"), **out)


def grid_small():
    """Grid2d (BASELINE config 3 generator, grid2d.py:40-89) at 13 x 9."""
    G = graphs.Grid2d(13, 9)
    out = csr_parts("W", G.W)
    out.update(lap_parts("g", G.W))
    G.estimate_lmax()
    out["lmax"] = np.float64(G.lmax)
    g = filters.MexicanHat(G, Nf=6)
    x = np.random.default_rng(0).standard_normal((G.N, 4))
    out["signal"] = x
    out["coeff"] = np.array(approximations.compute_cheby_coeff(g, m=50))
    out["filtered"] = g.filter(x, order=50)
    np.savez_compressed(os.path.join(HERE, "grid13x9.npz"), **out)


if __name__ == "__main__":
    print("pygsp", pygsp.__version__)
    logo()
    sensor123()
    doctest_027649()
    laplacian_kats()
    grid_small()
    for f in sorted(os.listdir(HERE)):
        if f.endswith(".npz"):
            print(f, os.path.getsize(os.path.join(HERE, f)))
