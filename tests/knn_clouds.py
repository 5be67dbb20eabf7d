"""Point clouds on which a cell-grid k-NN search can go wrong, shared by test_knn_grid_cpu.py (grid
sizing and binning, no GPU) and test_knn_grid_gpu.py (the search against the exhaustive one).

Tied lattices whose cell faces fall on lattice lines (so that ties sit exactly on the stopping
radius), duplicated points, degenerate and near-degenerate boxes (lines, planes, one or two
locations, spreads at rounding level), clusters with far outliers, and points on the box's
maximum faces.  n <= 20 000: even a cloud that ends up in one cell costs at most 4e8 distances.
"""
import functools
import zlib

import numpy as np

from pygsp_b200.graphs.generators import _knn_grid_cells


def _lattice(side, dim):
    axes = np.meshgrid(*[np.arange(float(side))] * dim, indexing="ij")
    return np.stack(axes, -1).reshape(-1, dim)


def face_ppc(X):
    """The first points_per_cell of 1, 1.25, ..., 15.75 for which every cell of the grid over the
    integer cloud X is an integer number of lattice steps wide: cell faces on lattice lines."""
    lo, hi = X.min(axis=0), X.max(axis=0)
    for ppc in np.arange(1.0, 16.0, 0.25):
        cells = _knn_grid_cells(lo, hi, X.shape[0], ppc)
        h = (hi - lo) / cells
        if (h > 1).all() and (h == np.round(h)).all():
            return float(ppc)
    raise AssertionError("no points_per_cell puts the faces on lattice lines")


def _shuffle(rng, X):
    return X[rng.permutation(X.shape[0])]


def _build(name):
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    if name.startswith("lattice"):
        dim = 2 if "2d" in name else 3
        X = _lattice(31 if dim == 2 else 21, dim)
        ppc = face_ppc(X)
        if "perm" in name:
            X = _shuffle(rng, X)
        if "shift" in name:
            X = X * 0.1 + 1e6
        return X, ppc
    if name == "repeat5":          # m = 5 copies: fewer than k + 1 for k = 10, 32, more for k = 1
        return _shuffle(rng, np.repeat(rng.integers(0, 40, (400, 2)).astype(float), 5, axis=0)), 3.0
    if name == "repeat40":         # m = 40 copies: more than k + 1 for every k <= 32
        return _shuffle(rng, np.repeat(rng.integers(-9, 9, (120, 3)).astype(float), 40, axis=0)), 3.0
    if name == "identical":
        return np.tile([3.0, -2.0], (500, 1)), 3.0
    if name == "two_locations":
        return np.array([[1.0, 2.0, 3.0], [2.0, 4.0, 6.0]])[rng.integers(0, 2, 600)], 3.0
    if name == "line_x_2d":        # y constant
        return np.stack([rng.permutation(20000).astype(float), np.full(20000, 7.0)], 1), 3.0
    if name == "line_z_3d":
        z = rng.integers(-3000, 3000, 8000).astype(float)
        return np.stack([np.full(8000, 2.0), np.full(8000, -3.0), z], 1), 3.0
    if name == "diagonal_2d":
        t = rng.integers(0, 5000, 6000).astype(float)
        return np.stack([t, t], 1), 3.0
    if name == "plane_z_3d":
        xy = rng.integers(0, 100, (8000, 2)).astype(float)
        return np.concatenate([xy, np.full((8000, 1), 5.0)], 1), 3.0
    if name == "spread1e-9_2d":
        return np.stack([rng.uniform(size=20000), 0.5 + 1e-9 * rng.uniform(size=20000)], 1), 3.0
    if name == "spread1e-14_2d":
        return np.stack([rng.uniform(size=1000), 1e-14 * rng.uniform(size=1000)], 1), 3.0
    if name == "spread1e-14_3d":
        X = rng.uniform(size=(5000, 3))
        X[:, 1] = 1.0 + 1e-14 * rng.uniform(size=5000)
        return X, 3.0
    if name == "cluster_outliers":  # radius 1e-6 around the origin, five points ~1e3 away
        X = rng.normal(scale=3e-7, size=(20000, 2))
        X[:5] = rng.uniform(-1e3, 1e3, (5, 2))
        return _shuffle(rng, X), 3.0
    if name == "two_clusters":
        X = rng.normal(scale=1e-3, size=(10000, 3))
        X[5000:] += 1e4
        return _shuffle(rng, X), 3.0
    if name == "far_point":
        X = rng.uniform(size=(5000, 2))
        X[1234] = [1e6, 1e6]
        return X, 3.0
    if name == "box_max":          # a lattice corner and face rows exactly at the maximum
        X = rng.integers(0, 30, (3000, 2)).astype(float)
        X[:40] = 30.0
        X[40:200, 0] = 30.0
        return _shuffle(rng, X), 3.0
    if name == "negative_3d":
        return rng.integers(-40, -10, (6000, 3)).astype(float), 3.0
    raise KeyError(name)


NAMES = ["lattice2d", "lattice2d_perm", "lattice3d", "lattice3d_perm", "lattice2d_perm_shift",
         "lattice3d_perm_shift", "repeat5", "repeat40", "identical", "two_locations",
         "line_x_2d", "line_z_3d", "diagonal_2d", "plane_z_3d", "spread1e-9_2d",
         "spread1e-14_2d", "spread1e-14_3d", "cluster_outliers", "two_clusters", "far_point",
         "box_max", "negative_3d"]


@functools.lru_cache(maxsize=None)
def _cached(name):
    X, ppc = _build(name)
    return np.ascontiguousarray(X, dtype=np.float64), ppc


def cloud(name):
    """(points (n, dim) float64, points_per_cell) of a named cloud, a fresh copy per call."""
    X, ppc = _cached(name)
    return X.copy(), ppc


def exact(X):
    """True when every squared distance of X is exact in float64 (small integer coordinates):
    then a NumPy brute force gives the true (distance, id) order."""
    return bool((X == np.round(X)).all() and np.abs(X).max() < 2 ** 20)
