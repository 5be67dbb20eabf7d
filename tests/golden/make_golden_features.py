"""Generate tests/golden/features.npz from the unmodified PyGSP 0.6.1 (CPU, NumPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_features.py

Contents (read by tests/test_oracle_features.py and tests/test_features_gpu.py):

  sensor_W_*           adjacency of graphs.Sensor(300, seed=42) (CSR parts)
  sensor_lmax          the reference's G.lmax (ARPACK estimate, unseeded: stored, not redone)
  spectr_default       features.compute_spectrogram(G) (M = 100), (300, 100)
  spectr_atom          features.compute_spectrogram(G, atom, M=20) with
                       atom(x) = 1 / (1 + (10 x / lmax)^2), (300, 20)
  norm_heat            features.compute_norm_tig(filters.Heat(G, scale=10)), (300,)
  norm_mh              features.compute_norm_tig(filters.MexicanHat(G, Nf=3)): the list of 3
                       (900,) arrays, stacked (3, 900)
  adj_<g>_W_*, adj_<g> features.compute_avg_adj_deg for g in sensor, directed (a directed
                       graph with self-loops and one negative weight), isolated (a graph with an
                       isolated vertex); the reference's np.matrix (N, 1) as an ndarray
"""
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "features.npz")


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def adjacency_cases():
    # directed: asymmetric random weights, self-loops on 5 vertices, one negative weight
    D = sparse.random(60, 60, density=0.08, random_state=3, format="lil")
    for v in (0, 7, 19, 33, 59):
        D[v, v] = 1.0 + v
    D[2, 5] = -0.5
    # isolated vertex 11 in a random symmetric graph
    S = sparse.random(40, 40, density=0.1, random_state=4, format="lil")
    S[11, :] = 0
    S[:, 11] = 0
    S = S + S.T
    S.setdiag(0)
    return {"directed": sparse.csr_matrix(D), "isolated": sparse.csr_matrix(S)}


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    from pygsp import features, filters, graphs
    logging.disable(logging.CRITICAL)
    out = {}
    G = graphs.Sensor(300, seed=42)
    G.estimate_lmax()
    lmax = float(G.lmax)
    out.update(csr_parts("sensor_W", G.W))
    out["sensor_lmax"] = np.float64(lmax)
    out["spectr_default"] = features.compute_spectrogram(G)
    out["spectr_atom"] = features.compute_spectrogram(
        G, atom=lambda x: 1.0 / (1.0 + (10.0 * x / lmax) ** 2), M=20)
    out["norm_heat"] = features.compute_norm_tig(filters.Heat(G, scale=10))
    mh = features.compute_norm_tig(filters.MexicanHat(G, Nf=3))
    assert isinstance(mh, list) and len(mh) == 3 and all(v.shape == (900,) for v in mh)
    out["norm_mh"] = np.stack(mh)
    out["adj_sensor"] = np.asarray(features.compute_avg_adj_deg(G))
    out.update(csr_parts("adj_sensor_W", G.W))
    for name, W in adjacency_cases().items():
        Gw = graphs.Graph(W)
        out["adj_" + name] = np.asarray(features.compute_avg_adj_deg(Gw))
        out.update(csr_parts("adj_%s_W" % name, Gw.W))
    np.savez_compressed(OUT, **out)
    print("%s: %d arrays, %d bytes" % (OUT, len(out), os.path.getsize(OUT)))


if __name__ == "__main__":
    main()
