"""Generate tests/golden/sampled_models.npz from the unmodified PyGSP 0.6.1 (CPU, SciPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_sampled_models.py

Contents (read by tests/test_sampled_models_cpu.py, tests/test_oracle_sampled_models.py and
tests/test_sampled_models_gpu.py):

  cases                   the names <g> of every graph below
  <g>_args                JSON {"model": class name, "kwargs": constructor arguments}
  <g>_W_*                 strict upper triangle of the adjacency (CSR parts: indptr, indices,
                          data as float64, shape); every W here is symmetric with a zero
                          diagonal, so W = T + T^T.  SwissRoll stores no data (see below)
  <g>_W_sha256            SwissRoll: SHA-256 of the float64 bytes of the triangle's data in CSR
                          order.  The weights are exp(-distanz(coords)^2 / 2 s^2), which
                          oracle/sampled_models_oracle.swissroll_reference restates; the CPU
                          tests check that restatement against this digest
  <g>_coords_sha256       SHA-256 of G.coords (float64, C order).  Coordinates are host NumPy
                          draws that must be equal bit for bit, so a digest is the whole check
                          and keeps the fixture small
  <g>_info_*              Community: node_com, comm_sizes, world_rad, com_coords
  <g>_info_json           Community: the scalar entries of G.info
  <g>_x_sha256            SwissRoll: SHA-256 of G.x
  <g>_labels              TwoMoons: G.labels
  <g>_layout_sha256       Community: SHA-256 of G.coords after set_coordinates('community2D',
                          seed=7)
  blocks_<s>              (seeds, Nc, Nc) edge counts between communities a >= b of the sampled
                          case <s> for seeds blocks_<s>_seeds (one community layout per seed)
  blocks_<s>_args         JSON of the case's arguments (without the seed)
  errors                  JSON [[model, kwargs, exception type name], ...] of invalid arguments
"""
import hashlib
import json
import logging
import os
import sys

import numpy as np
from scipy import sparse

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "sampled_models.npz")
BLOCK_SEEDS = 200

CASES = {
    "community_default_s0": ("Community", dict(seed=0)),
    "community_default_s1": ("Community", dict(seed=1)),
    "community_default_s2": ("Community", dict(seed=2)),
    "community_sizes": ("Community", dict(N=250, Nc=3, comm_sizes=[50, 120, 80], seed=42)),
    "community_epsilon": ("Community", dict(N=300, epsilon=2.5, seed=3)),
    "community_exact": ("Community", dict(N=2000, world_density=0, seed=4)),
    "community_exact_small": ("Community", dict(N=400, Nc=5, world_density=0, seed=8)),
    "community_dense_world": ("Community", dict(N=60, Nc=3, world_density=0.5, seed=5)),
    "community_comm_density": ("Community", dict(N=120, Nc=4, comm_density=0.3, seed=6)),
    "community_knn_empty": ("Community", dict(N=400, Nc=4, k_neigh=5, world_density=0, seed=0)),
    "swissroll_400_3d": ("SwissRoll", dict(N=400, seed=0)),
    "swissroll_1000_3d": ("SwissRoll", dict(N=1000, seed=1)),
    "swissroll_400_2d": ("SwissRoll", dict(N=400, dim=2, seed=2)),
    "swissroll_1000_2d": ("SwissRoll", dict(N=1000, dim=2, seed=3)),
    "swissroll_noise": ("SwissRoll", dict(N=400, noise=True, seed=4)),
    "swissroll_classic": ("SwissRoll", dict(N=400, srtype="classic", seed=5)),
    "sphere_s0": ("Sphere", dict(seed=0)),
    "sphere_s1": ("Sphere", dict(nb_pts=500, seed=1)),
    "sphere_4d": ("Sphere", dict(nb_pts=200, nb_dim=4, seed=2)),
    "cube_3d_s0": ("Cube", dict(seed=0)),
    "cube_3d_s1": ("Cube", dict(nb_pts=500, seed=1)),
    "cube_2d": ("Cube", dict(nb_pts=200, nb_dim=2, seed=2)),
    "twomoons_s0": ("TwoMoons", dict(moontype="synthesized", seed=0)),
    "twomoons_s1": ("TwoMoons", dict(moontype="synthesized", N=301, seed=1)),
}

BLOCKS = {
    "default": dict(),
    "dense_world": dict(N=60, Nc=3, world_density=0.5),
    "comm_density": dict(N=120, Nc=4, comm_density=0.3),
}

ERRORS = [
    ("Community", dict(N=100, min_deg=2)),
    ("Community", dict(N=100, world_density=1.5)),
    ("Community", dict(N=100, world_density=-0.1)),
    ("Community", dict(N=100, Nc=5, min_comm=30)),
    ("Community", dict(N=100, Nc=3, comm_sizes=[50, 50])),
    ("Community", dict(N=100, Nc=2, comm_sizes=[50, 40])),
    ("Community", dict(N=100, comm_density=1.5)),
    ("Community", dict(N=100, k_neigh=-1)),
    ("Cube", dict(nb_dim=4)),
    ("Cube", dict(sampling="grid")),
    ("Sphere", dict(sampling="grid")),
    ("TwoMoons", dict(moontype="crescent")),
]


def digest(a):
    return np.array(hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes())
                    .hexdigest())


def triu_parts(prefix, M, data=True):
    """CSR parts of the strict upper triangle of a symmetric M with a zero diagonal."""
    M = sparse.csr_matrix(M).astype(np.float64)
    assert (M != M.T).nnz == 0 and not M.diagonal().any(), prefix
    T = sparse.triu(M, k=1).tocsr()
    T.sort_indices()
    out = {prefix + "_indptr": T.indptr.astype(np.int32),
           prefix + "_indices": T.indices.astype(np.int32),
           prefix + "_shape": np.array(T.shape, dtype=np.int64)}
    if data:
        out[prefix + "_data"] = T.data.astype(np.float64)
    else:
        out[prefix + "_sha256"] = digest(T.data)
    return out


def block_counts(G):
    """(Nc, Nc) edge counts between communities, a >= b, of a Community."""
    com = np.asarray(G.info["node_com"])
    coo = sparse.tril(sparse.csr_matrix(G.W), k=-1).tocoo()
    a, b = com[coo.row], com[coo.col]
    lo, hi = np.minimum(a, b), np.maximum(a, b)
    out = np.zeros((G.Nc, G.Nc), dtype=np.int64)
    np.add.at(out, (hi, lo), 1)
    return out


def main():
    if REF:
        sys.path.insert(0, REF)
    import pygsp
    from pygsp import graphs
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import sampled_models_oracle
    assert pygsp.__version__ == "0.6.1", pygsp.__version__
    logging.getLogger("pygsp").setLevel(logging.ERROR)
    out = {"cases": np.array(sorted(CASES))}
    for name, (model, kwargs) in sorted(CASES.items()):
        G = getattr(graphs, model)(**kwargs)
        for lg in list(logging.Logger.manager.loggerDict.values()):
            if isinstance(lg, logging.Logger) and lg.name.startswith("pygsp"):
                lg.setLevel(logging.ERROR)
        out[name + "_args"] = np.array(json.dumps({"model": model, "kwargs": kwargs}))
        out.update(triu_parts(name + "_W", G.W, data=model != "SwissRoll"))
        out[name + "_coords_sha256"] = digest(G.coords)
        if model == "SwissRoll":        # the restatement gives the reference's bits
            restated = sampled_models_oracle.swissroll_reference(G.coords, G.s, G.thresh)
            assert (restated != sparse.triu(sparse.csr_matrix(G.W), k=1)).nnz == 0, name
            assert str(digest(restated.data)) == str(out[name + "_W_sha256"]), name
        if model == "Community":
            for key in ("node_com", "comm_sizes", "world_rad", "com_coords"):
                out["%s_info_%s" % (name, key)] = np.asarray(G.info[key])
            scalars = {k: v for k, v in G.info.items()
                       if k not in ("node_com", "comm_sizes", "world_rad", "com_coords")}
            out[name + "_info_json"] = np.array(json.dumps(scalars))
            G.set_coordinates("community2D", seed=7)
            out[name + "_layout_sha256"] = digest(G.coords)
        elif model == "SwissRoll":
            out[name + "_x_sha256"] = digest(G.x)
        elif model == "TwoMoons":
            out[name + "_labels"] = G.labels
    for name, kwargs in BLOCKS.items():
        seeds = np.arange(BLOCK_SEEDS)
        out["blocks_" + name] = np.stack([block_counts(graphs.Community(seed=int(s), **kwargs))
                                          for s in seeds])
        out["blocks_%s_seeds" % name] = seeds
        out["blocks_%s_args" % name] = np.array(json.dumps(kwargs))
    errors = []
    for model, kwargs in ERRORS:
        try:
            getattr(graphs, model)(**kwargs)
            errors.append([model, kwargs, None])
        except Exception as exc:             # noqa: BLE001 - recording the type is the point
            errors.append([model, kwargs, type(exc).__name__])
    out["errors"] = np.array(json.dumps(errors))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(CASES), "cases")


if __name__ == "__main__":
    main()
