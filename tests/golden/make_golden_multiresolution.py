"""Generate tests/golden/multiresolution.npz from the unmodified PyGSP 0.6.1 (CPU, SciPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_multiresolution.py

Contents (read by tests/test_oracle_multiresolution.py and tests/test_multiresolution_gpu.py),
for g in s256 (graphs.Sensor(256, seed=7)), s1000 (graphs.Sensor(1000, seed=1)) and grid
(graphs.Grid2d(16, 12)):

  <g>_W_*        adjacency (CSR parts)
  <g>_V          the reference's eigenvector of the largest eigenvalue (G.U[:, -1] after
                 compute_fourier_basis), times sign(V[0]) as graph_multiresolution does
  <g>_ind        np.nonzero(V >= 0)[0], the kept vertices
  <g>_kronW_*    reduction.kron_reduction(G, ind).W (Graph branch)
  <g>_kreg_*     reduction.kron_reduction(G.L + 0.005 I, ind) (matrix branch)

and for the multiresolution of graphs.Grid2d(20, 15) (reduction.graph_multiresolution(G, 3,
sparsify=False)):

  mr_levels      3
  mr_W<i>_*      adjacency of level i (i = 0..3)
  mr_idx<i>      Gs[i].mr['idx'] (i = 1..3)
  mr_Kreg<i>_*   Gs[i].mr['K_reg'] (i = 0..2)

The script checks that no fixture reaches the reference's Snew correction (reduction.py:366-369:
||Snew|| >= spacing(1000)), whose broadcast the device engine deliberately does not reproduce,
and that no |V_i| lies within 1e-8 max|V| of zero, so that ind is well defined -- except for
s1000: the largest eigenvector of a k-NN sensor graph is localised (on Sensor(1000, seed=s),
s = 1..12, min|V_i| / max|V| is below 5e-15), so the signs of its smallest entries are
round-off.  Its kron fixtures use the recorded ind as given; <g>_ambiguous counts the entries
with |V_i| <= 1e-8 max|V|.  The multiresolution fixture is a grid, whose levels all pass.
"""
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "multiresolution.npz")


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    M.sum_duplicates()
    M.sort_indices()
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def check_snew(L, ind, reduction):
    """Norm of the reference's Snew for the Graph branch of kron_reduction(G, ind)."""
    Lnew = reduction.kron_reduction(sparse.csr_matrix(L), ind)
    Wnew = sparse.diags(Lnew.diagonal(), 0) - Lnew
    Snew = Lnew.diagonal() - np.ravel(Wnew.sum(0))
    norm = np.linalg.norm(Snew, 2)
    assert norm < np.spacing(1000), norm
    return norm


def check_v(V):
    assert np.abs(V).min() > 1e-8 * np.abs(V).max(), np.abs(V).min()


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    from pygsp import graphs, reduction
    logging.disable(logging.CRITICAL)
    out = {}
    cases = {"s256": graphs.Sensor(256, seed=7), "s1000": graphs.Sensor(1000, seed=1),
             "grid": graphs.Grid2d(16, 12)}
    for name, G in cases.items():
        G.compute_fourier_basis()
        V = G.U[:, -1].copy()
        V *= np.sign(V[0])
        if name != "s1000":
            check_v(V)
        out[name + "_ambiguous"] = np.int64((np.abs(V) <= 1e-8 * np.abs(V).max()).sum())
        ind = np.nonzero(V >= 0)[0]
        print(name, "N", G.N, "kept", ind.size, "Snew", check_snew(G.L, ind, reduction))
        out.update(csr_parts(name + "_W", G.W))
        out[name + "_V"] = V
        out[name + "_ind"] = ind.astype(np.int64)
        out.update(csr_parts(name + "_kronW", reduction.kron_reduction(G, ind).W))
        out.update(csr_parts(name + "_kreg", reduction.kron_reduction(
            G.L + 0.005 * sparse.eye(G.N), ind)))

    G = graphs.Grid2d(20, 15)
    levels = 3
    Gs = reduction.graph_multiresolution(G, levels, sparsify=False)
    out["mr_levels"] = np.int64(levels)
    for i, g in enumerate(Gs):
        out.update(csr_parts("mr_W%d" % i, g.W))
        if i > 0:
            out["mr_idx%d" % i] = np.asarray(g.mr["idx"], dtype=np.int64)
        if i < levels:
            out.update(csr_parts("mr_Kreg%d" % i, g.mr["K_reg"]))
            g.compute_fourier_basis()
            V = g.U[:, -1].copy()
            V *= np.sign(V[0])
            check_v(V)
            assert np.array_equal(np.nonzero(V >= 0)[0], Gs[i + 1].mr["idx"])
            check_snew(g.L, Gs[i + 1].mr["idx"], reduction)
        print("level", i, "N", g.N, "nnz", g.W.nnz)
    np.savez_compressed(OUT, **out)
    print("%s: %d arrays, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
