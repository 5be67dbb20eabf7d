"""The cell grid of the device k-NN search (graphs.knn_device -> gsp_knn_grid), without a GPU:
how _knn_grid_cells sizes the grid on degenerate, clustered and tied clouds (tests/knn_clouds.py),
and where the kernel's binning puts every point relative to the cell faces its stopping test
measures to."""
import math
from fractions import Fraction

import numpy as np
import pytest

import knn_clouds
from pygsp_b200.graphs.generators import _knn_grid_cells

AXIS_MAX = 2 ** 30        # cells per axis that gsp_knn_grid accepts
CELLS_PER_POINT = 4
# The stopping test of knn_query_kernel (csrc/generate.cu) keeps slack = 2^-44 max(|lo|, |hi|)
# per axis and grants binning and face rounding together 1/16 of it.
BINNING_TOL = 2.0 ** -48


def _check_cells(cells, n):
    assert cells.dtype == np.int32
    assert (cells >= 1).all() and (cells <= AXIS_MAX).all(), cells
    total = math.prod(int(c) for c in cells)
    assert total < 2 ** 31 and total <= CELLS_PER_POINT * n, (cells, n)


@pytest.mark.parametrize("name", knn_clouds.NAMES)
def test_grid_size_of_every_cloud(name):
    X, ppc = knn_clouds.cloud(name)
    n = X.shape[0]
    lo, hi = X.min(axis=0), X.max(axis=0)
    cells = _knn_grid_cells(lo, hi, n, ppc)
    _check_cells(cells, n)
    span = hi - lo
    assert (cells[span <= 1e-6 * span.max()] == 1).all(), cells      # degenerate axes
    if np.count_nonzero(span) == 1:                                   # an axis-aligned line
        assert abs(int(cells[span > 0][0]) - n / ppc) <= 1, cells


@pytest.mark.parametrize("lo,hi,n,want", [
    ([0, 5], [1, 5], 1000, [333, 1]),                   # y constant: a zero span
    ([0, 0, 2], [1, 1, 2], 1000, [18, 18, 1]),          # a z = const plane
    ([3, 3], [3, 3], 50, [1, 1]),                       # every point identical
    ([0, 0], [1, 1e-14], 1000, [333, 1]),               # y spread far below one cell
    ([0, 0, 0], [1, 1e-9, 1], 20000, [81, 1, 81]),
    ([0, 0, 0], [1e-300, 1e-300, 1e-300], 10 ** 6, [69, 69, 69]),   # the volume underflows
    ([0, 0], [1, 1], 10 ** 6, [577, 577]),              # the Sensor(10^6) square
])
def test_grid_size_of_degenerate_boxes(lo, hi, n, want):
    cells = _knn_grid_cells(np.array(lo, dtype=float), np.array(hi, dtype=float), n, 3.0)
    _check_cells(cells, n)
    assert cells.tolist() == want


def test_grid_size_bounds():
    # a line of 2^31 - 1 points at 0.5 per cell asks for 4.3e9 cells along x
    assert _knn_grid_cells([0.0, 0.0], [1.0, 0.0], 2 ** 31 - 1, 0.5).tolist() == [AXIS_MAX, 1]
    # 1000 points, 1e-3 per cell: a million cells asked for, at most 4 per point kept
    cells = _knn_grid_cells([0.0, 0.0], [1.0, 1.0], 1000, 1e-3)
    _check_cells(cells, 1000)
    with pytest.raises(ValueError):
        _knn_grid_cells([-1e308, 0.0], [1e308, 1.0], 100, 3.0)        # the span overflows
    with pytest.raises(ValueError):
        _knn_grid_cells([0.0, 0.0], [np.inf, 1.0], 100, 3.0)
    with pytest.raises(ValueError):
        _knn_grid_cells([0.0, 0.0], [1.0, 1.0], 100, 0.0)


def test_grid_size_of_random_boxes():
    """Boxes whose spans run over 600 decades, zero included, any n and density."""
    rng = np.random.default_rng(5)
    for _ in range(3000):
        dim = int(rng.integers(2, 4))
        n = int(rng.integers(2, 2 ** 31))
        lo = rng.normal(size=dim) * 10.0 ** rng.integers(-300, 300, dim)
        span = rng.uniform(size=dim) * 10.0 ** rng.integers(-300, 300, dim)
        span[rng.uniform(size=dim) < 0.2] = 0.0
        hi = lo + span
        if not np.isfinite(hi - lo).all():
            continue
        cells = _knn_grid_cells(lo, hi, n, float(rng.uniform(0.05, 50)))
        _check_cells(cells, n)
        assert (cells[hi - lo == 0] == 1).all()


def _binning(X, cells):
    """gsp_knn_grid's h and 1/h and cell_coord's bins, in IEEE double: NumPy rounds the
    subtraction and the product separately, as the kernel does (no FMA can join them)."""
    lo, hi = X.min(axis=0), X.max(axis=0)
    span = hi - lo
    h = np.where(span > 0, span / cells, 1.0)
    c = np.floor((X - lo) * (1.0 / h))
    return lo, hi, h, np.clip(c, 0, cells - 1).astype(np.int64)


@pytest.mark.parametrize("name", knn_clouds.NAMES)
def test_binning_stays_within_the_stopping_margin(name):
    """A point in cell c lies above the face lo + c h and below lo + (c + 1) h but for the
    rounding the stopping test allows for, in exact arithmetic."""
    X, ppc = knn_clouds.cloud(name)
    cells = _knn_grid_cells(X.min(axis=0), X.max(axis=0), X.shape[0], ppc)
    lo, hi, h, c = _binning(X, cells)
    crossed = 0
    for d in range(X.shape[1]):
        tol = Fraction(BINNING_TOL * max(abs(lo[d]), abs(hi[d])))
        L, H = Fraction(lo[d]), Fraction(h[d])
        for x, cd in np.unique(np.stack([X[:, d], c[:, d]], axis=1), axis=0):
            x, cd = Fraction(x), int(cd)
            if cd > 0:
                assert x >= L + cd * H - tol, (name, d, x, cd)
                crossed += x < L + cd * H
            if cd < cells[d] - 1:
                assert x <= L + (cd + 1) * H + tol, (name, d, x, cd)
                crossed += x >= L + (cd + 1) * H
    if name.endswith("_shift"):
        # faces a rounding away from lattice lines: some points are binned across one, which
        # is why the stopping test needs its margin
        assert crossed > 0


def test_lattice_faces_fall_on_lattice_lines():
    """The lattices put ties exactly on the stopping radius: every cell is a whole number of
    lattice steps wide, and the 31 x 31 lattice gets the 15 x 15 grid of width 2."""
    for name in ("lattice2d", "lattice3d"):
        X, ppc = knn_clouds.cloud(name)
        lo, hi = X.min(axis=0), X.max(axis=0)
        h = (hi - lo) / _knn_grid_cells(lo, hi, X.shape[0], ppc)
        assert (h == np.round(h)).all() and (h > 1).all()
    X, ppc = knn_clouds.cloud("lattice2d")
    assert _knn_grid_cells(X.min(axis=0), X.max(axis=0), X.shape[0], ppc).tolist() == [15, 15]
