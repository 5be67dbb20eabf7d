"""Generate tests/golden/lanczos.npz from the unmodified PyGSP 0.6.1 (CPU, NumPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_lanczos.py

``lanczos_op`` (approximations.py:228-278) reads ``f.g``, which 0.6.1's Filter no longer has:
the script sets ``f.g = f._kernels`` on the filter object before the call, the one attribute
the function reads.  Contents (read by tests/test_oracle_lanczos.py and
tests/test_lanczos_gpu.py):

  graphs               names of the graphs: logo, sensor (Sensor(123, seed=42)), ring (Ring(64))
  <g>_W_*, <g>_L_*     adjacency and combinatorial Laplacian (CSR parts)
  <g>_lmax             G.lmax = the largest eigenvalue (the kernels below use it)
  <g>_x                seeded start vector of lanczos, (N,)
  <g>_V<o>, <g>_H<o>, <g>_orth<o>   lanczos(L.toarray(), o, x) for o in 1, 2, 20
  <g>_s1, <g>_s3       seeded signals (N,) and (N, 3), for g in logo, sensor
  <g>_<f>_<s>_o<o>     lanczos_op(f, s, order=o) for f in heat (Heat(scale=[5, 20])) and step
                       (Filter(G, lambda x: (x <= 0.3 * lmax) * 1.0)), s in s1, s3, o in 1, 10, 30
  <g>_<f>_<s>_exact    the exact filter output in the same layout, U f(Lambda) U^T s
"""
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "lanczos.npz")
ORDERS_BASIS = (1, 2, 20)
ORDERS_OP = (1, 10, 30)


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    from pygsp import filters, graphs
    from pygsp.filters import approximations
    logging.disable(logging.CRITICAL)
    out = {}
    made = {"logo": graphs.Logo(), "sensor": graphs.Sensor(123, seed=42), "ring": graphs.Ring(64)}
    out["graphs"] = np.array(list(made))
    rng = np.random.default_rng(11)
    for name, G in made.items():
        G.compute_fourier_basis()                     # sets G.lmax = e[-1], which Heat reads
        lmax = float(G.lmax)
        out.update(csr_parts(name + "_W", G.W))
        out.update(csr_parts(name + "_L", G.L))
        out[name + "_lmax"] = np.float64(lmax)
        x = rng.standard_normal(G.N)
        out[name + "_x"] = x
        for o in ORDERS_BASIS:
            V, H, orth = approximations.lanczos(G.L.toarray(), o, x)
            out["%s_V%d" % (name, o)] = V
            out["%s_H%d" % (name, o)] = H
            out["%s_orth%d" % (name, o)] = orth
        if name == "ring":
            continue
        s1, s3 = rng.standard_normal(G.N), rng.standard_normal((G.N, 3))
        out[name + "_s1"], out[name + "_s3"] = s1, s3
        bank = {"heat": filters.Heat(G, scale=[5, 20]),
                "step": filters.Filter(G, lambda x: (x <= 0.3 * lmax) * 1.0)}
        for fname, f in bank.items():
            f.g = f._kernels                          # the attribute lanczos_op reads (:247)
            fe = f.evaluate(G.e)                      # (Nf, N)
            for sname, s in (("s1", s1), ("s3", s3)):
                S = s.reshape(G.N, -1)
                exact = np.concatenate([G.U @ (fe[i][:, None] * (G.U.T @ S))
                                        for i in range(fe.shape[0])])
                key = "%s_%s_%s" % (name, fname, sname)
                out[key + "_exact"] = exact.reshape(-1) if s.ndim == 1 else exact
                for o in ORDERS_OP:
                    out["%s_o%d" % (key, o)] = approximations.lanczos_op(f, s, order=o)
    np.savez_compressed(OUT, **out)
    print("%s: %d arrays, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
