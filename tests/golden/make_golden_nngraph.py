"""Generate tests/golden/nngraph.npz from the unmodified PyGSP 0.6.1 (CPU, SciPy path).

    PYGSP_REFERENCE=<PyGSP 0.6.1 source tree> python tests/golden/make_golden_nngraph.py

The reference's patch graphs call skimage.util.view_as_windows; scikit-image is not needed: for
the run a stand-in module built on numpy's sliding_window_view (the same view for step 1) is put
into sys.modules, and the reference's own padding and reshape produce the features.

Contents (read by tests/test_oracle_nngraph.py and tests/test_nngraph_gpu.py):

  X_d<d>                 seeded normal cloud, 60 x d, for d in DIMS
  eps_d<d>_<metric>      the radius used with that cloud and metric (midway between two
                         consecutive pairwise distances, so that no pair lies near the boundary)
  nn_<type>_d<d>_<metric>_<sym>_W_*, ..._sigma
                         graphs.NNGraph(X, NNtype=type, dist_type=..., symmetrize_type=sym)
                         for type in {knn, radius}, every metric (minkowski with order 3) and
                         every symmetrize_type; W as canonical CSR parts
  img_gray, img_rgb      seeded uniform images, 16 x 12 and 9 x 11 x 3
  ip_<img>_<shape>_W_*, ..._sigma, ..._X
                         graphs.ImgPatches(img, patch_shape) (shape tag 3x3, 4x2, 5) and its
                         features Xin
  g2ip_<img>_<shape>_W_* graphs.Grid2dImgPatches(img, patch_shape=...) (default aggregate)
"""
import logging
import os
import sys
import types

import numpy as np
from scipy import sparse
from scipy.spatial import distance

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYGSP_REFERENCE") or (sys.argv[1] if len(sys.argv) > 1 else None)
OUT = os.path.join(HERE, "nngraph.npz")

DIMS = (1, 3, 8, 27)
METRICS = {"euclidean": 2.0, "manhattan": 1.0, "max_dist": np.inf, "minkowski": 3.0}
SYMS = ("average", "maximum", "fill", "tril", "triu")
PATCH_SHAPES = {"3x3": (3, 3), "4x2": (4, 2), "5": (5,)}
N_POINTS = 60


def csr_parts(prefix, M):
    M = sparse.csr_matrix(M)
    M.sum_duplicates()
    M.eliminate_zeros()
    M.sort_indices()
    return {prefix + "_indptr": M.indptr.astype(np.int32),
            prefix + "_indices": M.indices.astype(np.int32),
            prefix + "_data": M.data.astype(np.float64),
            prefix + "_shape": np.array(M.shape, dtype=np.int64)}


def install_skimage_standin():
    util = types.ModuleType("skimage.util")

    def view_as_windows(arr_in, window_shape, step=1):
        assert step == 1
        return np.lib.stride_tricks.sliding_window_view(arr_in, window_shape)

    util.view_as_windows = view_as_windows
    mod = types.ModuleType("skimage")
    mod.util = util
    sys.modules["skimage"] = mod
    sys.modules["skimage.util"] = util


def prepared(X):
    """The reference's center + rescale (nngraph.py:127-136) of a copy of X."""
    N, d = X.shape
    Y = X - np.mean(X, axis=0)
    radius = 0.5 * np.linalg.norm(Y.max(axis=0) - Y.min(axis=0), 2)
    return Y * ((np.power(N, 1.0 / float(min(d, 3))) / 10.0) / radius)


def radius_for(X, p, per_point=4):
    """A radius with about per_point neighbours per point, midway between two distances."""
    D = np.sort(distance.pdist(prepared(X), "minkowski", p=p))
    m = min(len(D) - 2, per_point * X.shape[0] // 2)
    return 0.5 * (D[m] + D[m + 1])


def main():
    if not REF:
        raise SystemExit(__doc__)
    sys.path.insert(0, REF)
    install_skimage_standin()
    from pygsp import graphs
    logging.disable(logging.CRITICAL)
    out = {}
    rng = np.random.default_rng(2024)
    for d in DIMS:
        X = rng.normal(size=(N_POINTS, d))
        out["X_d%d" % d] = X
        for metric, p in METRICS.items():
            eps = radius_for(X, p)
            out["eps_d%d_%s" % (d, metric)] = np.float64(eps)
            extra = {"order": 3} if metric == "minkowski" else {}
            for nntype in ("knn", "radius"):
                for sym in SYMS:
                    G = graphs.NNGraph(X.copy(), NNtype=nntype, dist_type=metric, epsilon=eps,
                                       symmetrize_type=sym, **extra)
                    tag = "nn_%s_d%d_%s_%s" % (nntype, d, metric, sym)
                    out.update(csr_parts(tag + "_W", G.W))
                    out[tag + "_sigma"] = np.float64(G.sigma)
    images = {"gray": rng.uniform(size=(16, 12)), "rgb": rng.uniform(size=(9, 11, 3))}
    for name, img in images.items():
        out["img_" + name] = img
        for tag, shape in PATCH_SHAPES.items():
            G = graphs.ImgPatches(img.copy(), patch_shape=shape)
            out.update(csr_parts("ip_%s_%s_W" % (name, tag), G.W))
            out["ip_%s_%s_sigma" % (name, tag)] = np.float64(G.sigma)
            out["ip_%s_%s_X" % (name, tag)] = np.asarray(G.Xin, dtype=np.float64)
            G2 = graphs.Grid2dImgPatches(img.copy(), patch_shape=shape)
            out.update(csr_parts("g2ip_%s_%s_W" % (name, tag), G2.W))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, len(out), "arrays")


if __name__ == "__main__":
    main()
