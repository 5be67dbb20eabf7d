"""Generate tests/golden/connectivity.npz from the unmodified PyGSP 0.6.1 (CPU, SciPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_connectivity.py

Contents (read by tests/test_oracle_connectivity.py and tests/test_connectivity_gpu.py), for every
graph <g> of GRAPHS:

  <g>_W_*                 adjacency (CSR parts: indptr, indices, data, shape)
  <g>_directed            G.is_directed()                                  (graph.py:368-405)
  <g>_connected           G.is_connected()                                 (:294-366)
  <g>_weighted            G.is_weighted()                                  (:257-292)

and, for an undirected graph, its G.extract_components() (:444-508):

  <g>_n_components        number of components
  <g>_comp<k>_orig_idx    component k's info['orig_idx'] (int64)
  <g>_comp<k>_W_*         component k's adjacency, canonical CSR parts

For the subgraph cases <s> of SUBGRAPHS, on graph <g> = <s>_graph with coords <g>_coords and a
signal 'sig' = <g>_signal attached by set_signal (:192-216), G.subgraph(<s>_sel) (:218-255):

  <s>_sel                 the selection as passed (an index list or a boolean mask)
  <s>_W_*, <s>_coords, <s>_signal   the subgraph's adjacency, coords and signals['sig']
"""
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_difference import csr_parts, directed_loops  # noqa: E402

REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "connectivity.npz")


def islands(n=60, seed=3):
    """Seeded sparse symmetric random graph: several components and isolated vertices."""
    rng = np.random.default_rng(seed)
    W = sparse.random(n, n, density=0.012, random_state=rng, format="csr")
    W = sparse.triu(W + W.T, k=1)
    W = (W + W.T).tocsr()
    W.data = 0.5 + W.data
    return W


def graphs_of(graphs):
    doc = [[0, 3, 0, 0], [3, 0, 4, 0], [0, 4, 0, 2], [0, 0, 2, 0]]     # graph.py:318-336, 234-244
    return {
        # test_graphs.py:136-172
        "ic_undirected": graphs.Graph([[0, 1, 0], [1, 0, 2], [0, 2, 0]]),
        "ic_directed_split": graphs.Graph([[0, 1, 0], [1, 0, 0], [0, 2, 0]]),
        "ic_undirected_split": graphs.Graph([[0, 1, 0], [1, 0, 0], [0, 0, 0]]),
        "ic_directed_cycle": graphs.Graph([[0, 1, 0], [0, 0, 2], [3, 0, 0]]),
        "doc_connected": graphs.Graph(doc),
        "doc_disconnected": graphs.Graph([[0, 3, 0, 0], [3, 0, 4, 0], [0, 0, 0, 2],
                                          [0, 0, 2, 0]]),
        "doc_binary": graphs.Graph([[0, 1, 0], [1, 0, 1], [0, 1, 0]]),       # :273-289
        "doc_weighted": graphs.Graph([[0, 2, 0], [2, 0, 1], [0, 1, 0]]),
        "negative": graphs.Graph([[0, 3, 0, 0], [3, 0, -4, 0], [0, -4, 0, 2], [0, 0, 2, 0]]),
        "logo": graphs.Logo(),
        "sensor": graphs.Sensor(123, seed=42),
        "er": graphs.ErdosRenyi(98, p=0.015, directed=False, seed=42),
        "er_directed": graphs.ErdosRenyi(98, p=0.015, directed=True, seed=42),
        "islands": graphs.Graph(islands()),
        "zeros": graphs.Graph(np.zeros((11, 11))),
        "identity": graphs.Graph(np.identity(11)),
        "random_loops": graphs.Graph(directed_loops()),
    }


def subgraphs_of(rng):
    n = 123
    return {
        "sub_sorted": ("sensor", np.sort(rng.choice(n, 60, replace=False))),
        "sub_unsorted": ("sensor", rng.choice(n, 50, replace=False)),
        "sub_repeats": ("sensor", np.array([5, -1, 5, 17, -123, 40, 17, 0, 121, -2])),
        "sub_mask": ("sensor", rng.random(n) < 0.4),
        "sub_empty": ("sensor", np.zeros(0, dtype=np.int64)),
        "sub_doc": ("doc_connected", np.array([0, 2, 1])),                  # graph.py:234-244
    }


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    from pygsp import graphs
    logging.disable(logging.CRITICAL)
    all_graphs = graphs_of(graphs)
    out = {"graphs": np.array(sorted(all_graphs))}
    for name, G in sorted(all_graphs.items()):
        out.update(csr_parts(name + "_W", G.W))
        out[name + "_directed"] = np.bool_(G.is_directed())
        out[name + "_connected"] = np.bool_(G.is_connected())
        out[name + "_weighted"] = np.bool_(G.is_weighted())
        if G.is_directed():
            continue
        comps = G.extract_components()
        out[name + "_n_components"] = np.int64(len(comps))
        for k, C in enumerate(comps):
            p = "%s_comp%d" % (name, k)
            out[p + "_orig_idx"] = np.asarray(C.info["orig_idx"], dtype=np.int64)
            W = sparse.csr_matrix(C.W)
            assert W.has_canonical_format
            out.update(csr_parts(p + "_W", W))

    rng = np.random.default_rng(2024)
    cases = subgraphs_of(rng)
    out["subgraphs"] = np.array(sorted(cases))
    for gname in sorted({g for g, _ in cases.values()}):
        G = all_graphs[gname]
        n = G.n_vertices
        out[gname + "_coords"] = rng.uniform(size=(n, 2))
        out[gname + "_signal"] = rng.normal(size=(n, 3))
    for sname, (gname, sel) in sorted(cases.items()):
        G = all_graphs[gname]
        W = sparse.csr_matrix(G.W)
        G = graphs.Graph(W, coords=out[gname + "_coords"])
        G.set_signal(out[gname + "_signal"], "sig")
        S = G.subgraph(list(sel) if sel.dtype != bool else sel)
        out[sname + "_graph"] = np.array(gname)
        out[sname + "_sel"] = sel
        out.update(csr_parts(sname + "_W", S.W))
        out[sname + "_coords"] = np.asarray(S.coords, dtype=np.float64).reshape(-1, 2)
        out[sname + "_signal"] = np.asarray(S.signals["sig"], dtype=np.float64).reshape(-1, 3)
    np.savez_compressed(OUT, **out)
    print("%s: %d arrays, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
