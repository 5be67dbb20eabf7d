"""Generate tests/golden/layout.npz from the unmodified PyGSP 0.6.1 (CPU).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_layout.py

The spring runs call the reference's own ``_sparse_fruchterman_reingold`` (_layout.py:169-219)
on A = W > 0 and on copies of the start, which it updates in place.  Contents (read by
tests/test_oracle_layout.py and tests/test_layout_gpu.py):

  graphs                    the graph names below (one string per name)
  g_<name>_W_*              the adjacency as canonical CSR parts
  g_<name>_start            the start: default_rng(seed).uniform(size=(N, 2)) (duplicated rows
                            for 'dup')
  g_<name>_run<it>          the positions after it iterations from the start, it in RUNS
  g_<name>_step_<state>     one iteration (t = 0.1) from the state 'start', 'run10' or 'run50'
  sc_names                  the set_coordinates cases
  sc_<case>                 G.set_coordinates(kind, seed, **kwargs).coords of the reference
  sc_<case>_call            JSON: {"graph", "kind", "seed", "kwargs"}; a 'pos' keyword names
                            the array sc_<case>_pos
  sbm_node_com, sbm_comm_sizes, sbm_world_rad
                            the info of the 'sbm' graph, for 'community2D'

Graphs: Sensor(300), Grid2d(20), ErdosRenyi(500, p=0.02), a stochastic block model of 600
vertices, a directed W with negative weights and self-loops, a disconnected graph with isolated
vertices, a start with duplicate positions, and N = 1, 2 and 257.
"""
import json
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "layout.npz")
RUNS = (1, 2, 10, 50)


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    M.sum_duplicates()
    M.eliminate_zeros()
    M.sort_indices()
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def directed_w(rng, n):
    """Non-symmetric weights in [-1, 1), some self-loops of either sign."""
    W = sparse.random(n, n, density=0.05, random_state=rng, data_rvs=lambda m: rng.uniform(-1, 1, m))
    W = sparse.lil_matrix(W)
    for i in rng.choice(n, 12, replace=False):
        W[i, i] = rng.choice([-0.5, 0.7])
    return sparse.csr_matrix(W)


def disconnected_w(rng):
    """Two random blocks of 70 vertices and 10 isolated vertices (N = 150)."""
    blocks = []
    for _ in range(2):
        B = sparse.random(70, 70, density=0.06, random_state=rng)
        B = sparse.triu(B, 1)
        blocks.append(B + B.T)
    return sparse.csr_matrix(sparse.block_diag(blocks + [sparse.csr_matrix((10, 10))]))


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    from pygsp import graphs
    from pygsp.graphs import _layout
    logging.disable(logging.CRITICAL)
    rng = np.random.default_rng(2026)

    ref_graphs = {
        "sensor300": graphs.Sensor(300, seed=42),
        "grid": graphs.Grid2d(20),
        "er": graphs.ErdosRenyi(500, p=0.02, seed=3),
        "sbm": graphs.StochasticBlockModel(N=600, k=4, p=0.1, q=0.005, seed=4),
        "n257": graphs.Sensor(257, seed=5),
    }
    W = {name: G.W for name, G in ref_graphs.items()}
    W["directed"] = directed_w(rng, 120)
    W["disconnected"] = disconnected_w(rng)
    W["dup"] = graphs.ErdosRenyi(100, p=0.05, seed=6).W
    W["n1"] = sparse.csr_matrix((1, 1))
    W["n2"] = sparse.csr_matrix(np.array([[0.0, 1.0], [1.0, 0.0]]))

    out = {"graphs": np.array(sorted(W))}
    for s, name in enumerate(sorted(W)):
        n = W[name].shape[0]
        A = W[name] > 0
        start = np.random.default_rng(100 + s).uniform(size=(n, 2))
        if name == "dup":
            start[10:20] = start[0]
            start[51] = start[50]
        out.update(csr_parts("g_%s_W" % name, W[name]))
        out["g_%s_start" % name] = start
        for it in RUNS:
            out["g_%s_run%d" % (name, it)] = _layout._sparse_fruchterman_reingold(
                A, 2, None, start.copy(), [], it, None)
        for state in ("start", "run10", "run50"):
            out["g_%s_step_%s" % (name, state)] = _layout._sparse_fruchterman_reingold(
                A, 2, None, out["g_%s_%s" % (name, state)].copy(), [], 1, None)
        print(name, n, flush=True)

    G = ref_graphs["sensor300"]
    pos_fixed = 3.0 * np.random.default_rng(11).uniform(size=(G.N, 2))
    cases = {
        "line1D": ("sensor300", "line1D", None, {}),
        "line2D": ("sensor300", "line2D", None, {}),
        "ring2D": ("sensor300", "ring2D", None, {}),
        "random2D": ("sensor300", "random2D", 7, {}),
        "random3D": ("sensor300", "random3D", 7, {}),
        "eigenmap2D": ("sensor300", "laplacian_eigenmap2D", None, {}),
        "eigenmap3D": ("sensor300", "laplacian_eigenmap3D", None, {}),
        "community2D": ("sbm", "community2D", 9, {}),
        "spring": ("sensor300", "spring", 42, {}),
        "spring_dim1": ("sensor300", "spring", 1, {"dim": 1, "iterations": 10}),
        "spring_dim3": ("sensor300", "spring", 2, {"dim": 3, "iterations": 10}),
        "spring_dim4": ("sensor300", "spring", 3, {"dim": 4, "iterations": 10}),
        "spring_fixed": ("sensor300", "spring", 4, {"pos": "pos", "fixed": [0, 5, 17],
                                                    "iterations": 10}),
        "spring_k": ("sensor300", "spring", 5, {"k": 0.2, "iterations": 10}),
        "spring_scale_center": ("sensor300", "spring", 6, {"scale": 2.5, "center": [[1.0, -2.0]],
                                                           "iterations": 10}),
        "spring_bad_center": ("sensor300", "spring", 7, {"center": [[1.0, 2.0, 3.0]],
                                                         "iterations": 10}),
        "spring_dir": ("directed", "spring", 8, {"iterations": 10}),
    }
    for case, (gname, kind, seed, kwargs) in cases.items():
        Gc = ref_graphs.get(gname) or graphs.Graph(W[gname])
        kw = dict(kwargs)
        if kw.get("pos") == "pos":
            kw["pos"] = pos_fixed.copy()
            out["sc_%s_pos" % case] = pos_fixed
        Gc.set_coordinates(kind, seed=seed, **kw)
        out["sc_" + case] = np.asarray(Gc.coords)
        out["sc_%s_call" % case] = np.array(json.dumps(
            {"graph": gname, "kind": kind, "seed": seed, "kwargs": kwargs}))
    out["sc_names"] = np.array(sorted(cases))
    sbm = ref_graphs["sbm"]
    out["sbm_node_com"] = np.asarray(sbm.info["node_com"])
    out["sbm_comm_sizes"] = np.asarray(sbm.info["comm_sizes"])
    out["sbm_world_rad"] = np.float64(sbm.info["world_rad"])
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
