"""Generate tests/golden/simplex.npz from the unmodified PyGSP 0.6.1 (CPU, NumPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_simplex.py

``classification_tikhonov_simplex`` (learning.py:42-180) imports pyunlocbox, which this project
does not depend on: the script installs oracle/unlocbox_standin.py in its place, so that the
reference's own function (projection, objective and gradient included) runs unchanged.
Contents (read by tests/test_oracle_simplex.py and tests/test_simplex_gpu.py):

  cases                names of the problems: logo (the reference's doctest: Logo(),
                       default_rng(42) mask > 0.5, tau 0.1), sensor and sensor10 (Sensor(123,
                       seed=42), 4 classes by quadrant, tau 0.1 and 10), ring (Ring(64), 2 classes)
                       and hand (a hand-built W: a path, a triangle with a pendant vertex and an
                       isolated vertex, 3 classes)
  <c>_W_*, <c>_L_*     adjacency and combinatorial Laplacian (CSR parts)
  <c>_lmax             G.lmax of the run (estimate_lmax for logo, the exact value otherwise)
  <c>_y, <c>_M, <c>_tau  the inputs (y is NaN where M is False)
  <c>_sol, <c>_niter, <c>_crit, <c>_obj   the default stop (rtol 1e-3, maxit 200): solution,
                       iteration count, criterion and objective f_0 .. f_niter
  <c>_sol<k>           the solution after exactly k iterations (rtol=None, maxit=k), k = 1, 2, 17
  <c>_conv             maxit=5000, rtol=None: the converged minimiser
"""
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "simplex.npz")
FIXED = (1, 2, 17)


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def hand_graph(graphs):
    edges = [(0, 1, 1.0), (1, 2, 2.0), (2, 3, 0.5), (4, 5, 1.0), (5, 6, 1.5), (4, 6, 1.0),
             (6, 7, 3.0)]
    W = np.zeros((9, 9))
    for i, j, w in edges:
        W[i, j] = W[j, i] = w
    return graphs.Graph(W)


def problems(graphs):
    out = []
    G = graphs.Logo()
    G.estimate_lmax()
    signal = np.zeros(G.n_vertices)
    signal[G.info["idx_s"]] = 1
    signal[G.info["idx_p"]] = 2
    rng = np.random.default_rng(42)
    mask = rng.uniform(0, 1, G.n_vertices) > 0.5
    measures = signal.copy()
    measures[~mask] = np.nan
    out.append(("logo", G, measures, mask, 0.1))

    G = graphs.Sensor(123, seed=42)
    G.compute_fourier_basis()
    xy = G.coords
    labels = (xy[:, 0] > np.median(xy[:, 0])) + 2 * (xy[:, 1] > np.median(xy[:, 1]))
    mask = np.random.default_rng(5).uniform(0, 1, G.n_vertices) > 0.6
    y = labels.astype(float)
    y[~mask] = np.nan
    out.append(("sensor", G, y, mask, 0.1))
    out.append(("sensor10", G, y, mask, 10.0))

    G = graphs.Ring(64)
    G.compute_fourier_basis()
    y = (np.arange(64) >= 32).astype(float)
    mask = np.zeros(64, dtype=bool)
    mask[[3, 20, 40, 55]] = True
    y[~mask] = np.nan
    out.append(("ring", G, y, mask, 0.1))

    G = hand_graph(graphs)
    G.compute_fourier_basis()
    y = np.array([0, np.nan, np.nan, 1, 2, np.nan, np.nan, 1, np.nan])
    mask = ~np.isnan(y)
    out.append(("hand", G, y, mask, 0.5))
    return out


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    sys.path.insert(0, ROOT)
    from oracle import unlocbox_standin
    unlocbox_standin.install()
    import pyunlocbox
    from pygsp import graphs, learning
    logging.disable(logging.CRITICAL)

    runs = {}
    real_solve = pyunlocbox.solvers.solve

    def recording_solve(*args, **kwargs):
        ret = real_solve(*args, **kwargs)
        runs["last"] = ret
        return ret
    pyunlocbox.solvers.solve = recording_solve

    out = {}
    cases = problems(graphs)
    out["cases"] = np.array([c[0] for c in cases])
    for name, G, y, M, tau in cases:
        out.update(csr_parts(name + "_W", G.W))
        out.update(csr_parts(name + "_L", G.L))
        out[name + "_lmax"] = np.float64(G.lmax)
        out[name + "_y"], out[name + "_M"], out[name + "_tau"] = y, M, np.float64(tau)
        sol = learning.classification_tikhonov_simplex(G, y, M, tau=tau, verbosity="NONE")
        ret = runs["last"]
        out[name + "_sol"] = np.asarray(sol)
        out[name + "_niter"] = np.int64(ret["niter"])
        out[name + "_crit"] = np.array(ret["crit"])
        out[name + "_obj"] = np.array([np.sum(o) for o in ret["objective"]])
        for k in FIXED:
            out["%s_sol%d" % (name, k)] = learning.classification_tikhonov_simplex(
                G, y, M, tau=tau, rtol=None, maxit=k, verbosity="NONE")
        out[name + "_conv"] = learning.classification_tikhonov_simplex(
            G, y, M, tau=tau, rtol=None, maxit=5000, verbosity="NONE")
        print(name, G.N, ret["niter"], ret["crit"])
    np.savez_compressed(OUT, **out)
    print("%s: %d arrays, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
