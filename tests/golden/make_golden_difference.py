"""Generate tests/golden/difference.npz from the unmodified PyGSP 0.6.1 (CPU, SciPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_difference.py

Contents (read by tests/test_oracle_difference.py and tests/test_difference_gpu.py), for every
graph <g> of GRAPHS:

  <g>_W_*                 adjacency (CSR parts: indptr, indices, data, shape)
  <g>_directed            G.is_directed()
  <g>_n_edges             G.n_edges
  <g>_sources / _targets / _weights   G.get_edge_list()                (graph.py:1019-1029)
  <g>_x, <g>_X            seeded vertex signal (N,) and block (N, 3), integers in [-4, 4]
  <g>_y, <g>_Y            seeded edge signal (Ne,) and block (Ne, 3), integers in [-4, 4]

and for each Laplacian type <t> in (combinatorial, normalized), after
G.compute_laplacian(<t>); G.compute_differential_operator():

  <g>_<t>_D_indptr / _indices / _data   CSC arrays of G.D               (difference.py:144-166)
  <g>_<t>_grad_x, _grad_X               G.grad(x), G.grad(X)            (difference.py:243-244)
  <g>_<t>_div_y, _div_Y                 G.div(y), G.div(Y)              (difference.py:325-331)
  <g>_<t>_energy_x, _energy_X           G.dirichlet_energy(x), (X)      (graph.py:701-702)
"""
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "difference.npz")
LAP_TYPES = ("combinatorial", "normalized")


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def directed_loops(n=40, seed=7):
    """Seeded random directed weighted graph with self-loops and one isolated vertex (n - 1)."""
    rng = np.random.default_rng(seed)
    W = sparse.random(n, n, density=0.12, random_state=rng, format="lil")
    W[n - 1, :] = 0
    W[:, n - 1] = 0
    for i in (0, 3, 11, 20):
        W[i, i] = 0.5 + i / 10
    W = sparse.csr_matrix(W)
    W.data = 0.1 + W.data
    return W


def graphs_of(graphs):
    return {
        "tri_undirected": graphs.Graph([[0, 2, 0], [2, 0, 1], [0, 1, 0]]),   # difference.py:94-110
        "tri_directed": graphs.Graph([[0, 2, 0], [2, 0, 1], [0, 0, 0]]),     # :114-130
        "edges_directed": graphs.Graph([[0, 3, 0], [3, 0, 4], [0, 0, 0]]),   # graph.py:997-1004
        "edges_undirected": graphs.Graph([[0, 3, 0], [3, 0, 4], [0, 4, 0]]),  # :1008-1015
        "path4": graphs.Path(4, directed=False),                            # difference.py:216-322
        "path4_directed": graphs.Path(4, directed=True),
        "path5": graphs.Path(5, directed=False),                            # graph.py:680-698
        "path5_directed": graphs.Path(5, directed=True),
        "logo": graphs.Logo(),
        "sensor": graphs.Sensor(123, seed=42),
        "er": graphs.ErdosRenyi(98, directed=False, seed=42),               # test_graphs.py:396-403
        "er_directed": graphs.ErdosRenyi(98, directed=True, seed=42),
        "small_directed": graphs.Graph([[1.3, 0], [0.4, 0.5]]),
        "zeros": graphs.Graph(np.zeros((11, 11))),                          # test_graphs.py:432-453
        "identity": graphs.Graph(np.identity(11)),
        "random_loops": graphs.Graph(directed_loops()),
    }


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    from pygsp import graphs
    logging.disable(logging.CRITICAL)
    out = {"graphs": np.array(sorted(graphs_of(graphs)))}
    for gi, (name, G) in enumerate(sorted(graphs_of(graphs).items())):
        rng = np.random.default_rng(100 + gi)
        out.update(csr_parts(name + "_W", G.W))
        out[name + "_directed"] = np.bool_(G.is_directed())
        out[name + "_n_edges"] = np.int64(G.n_edges)
        s, t, w = G.get_edge_list()
        out[name + "_sources"] = s.astype(np.int32)
        out[name + "_targets"] = t.astype(np.int32)
        out[name + "_weights"] = w.astype(np.float64)
        # small integers: exact in float32, and the fixture stays small (unit-weight graphs
        # then have integer or few-valued outputs, which compress)
        x, X = (rng.integers(-4, 5, size=sh).astype(np.float64) for sh in (G.N, (G.N, 3)))
        y, Y = (rng.integers(-4, 5, size=sh).astype(np.float64)
                for sh in (G.n_edges, (G.n_edges, 3)))
        out.update({name + "_x": x, name + "_X": X, name + "_y": y, name + "_Y": Y})
        for lap in LAP_TYPES:
            G.compute_laplacian(lap)
            G.compute_differential_operator()
            p = "%s_%s_" % (name, lap)
            D = G.D
            assert sparse.isspmatrix_csc(D) and D.has_canonical_format
            out[p + "D_indptr"] = D.indptr.astype(np.int32)
            out[p + "D_indices"] = D.indices.astype(np.int32)
            out[p + "D_data"] = D.data.astype(np.float64)
            out[p + "grad_x"], out[p + "grad_X"] = G.grad(x), G.grad(X)
            out[p + "div_y"], out[p + "div_Y"] = G.div(y), G.div(Y)
            out[p + "energy_x"] = np.float64(G.dirichlet_energy(x))
            out[p + "energy_X"] = np.asarray(G.dirichlet_energy(X), dtype=np.float64)
    np.savez_compressed(OUT, **out)
    print("%s: %d arrays, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
