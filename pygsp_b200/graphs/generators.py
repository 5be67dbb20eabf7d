"""Graph models that produce the inputs of the BASELINE configurations.

Each class builds an adjacency ``W`` and hands it to :class:`Graph`; what they
generate follows the reference generators (file:line cited per class) but the
construction is vectorised -- the reference's per-vertex Python loops
(nngraph.py:221-226) make it unusable beyond ~1e6 vertices.  They are input
fabrication for the filtering path, not part of the timed hot path.
"""
import math
import os

import numpy as np
from scipy import sparse, spatial

from .. import _native as nat
from .. import utils
from .csr import DeviceCSR, row_ids
from .graph import Graph, _torch_dtype

_DATA = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "data")


def morton_order(coords, bits=None):
    """Permutation that sorts points along a Z-order (Morton) curve.

    Vertex ids that are close in memory are then close in space, which is what
    makes the neighbour gather of the SpMM hit L1/L2 (SURVEY.md section 7,
    "gather locality").  Works for 2-D and 3-D coordinates.
    """
    coords = np.asarray(coords, dtype=np.float64)
    n, d = coords.shape
    if bits is None:
        bits = 21 if d <= 3 else 64 // d
    lo = coords.min(axis=0)
    span = np.maximum(coords.max(axis=0) - lo, 1e-300)
    q = np.minimum(((coords - lo) / span * (1 << bits)).astype(np.uint64), (1 << bits) - 1)
    code = np.zeros(n, dtype=np.uint64)
    for b in range(bits):
        for k in range(d):
            code |= ((q[:, k] >> np.uint64(b)) & np.uint64(1)) << np.uint64(b * d + k)
    return np.argsort(code, kind="stable")


class Logo(Graph):
    r"""GSP logo graph, N = 1130 (pygsp/graphs/logo.py:21-33).

    The adjacency and coordinates are the ones of the reference's
    ``data/pointclouds/logogsp.mat``, stored as ``pygsp_b200/data/logo.npz``.
    """

    def __init__(self, **kwargs):
        z = np.load(os.path.join(_DATA, "logo.npz"))
        n = len(z["indptr"]) - 1
        W = sparse.csr_matrix((z["data"], z["indices"], z["indptr"]), shape=(n, n))
        self.info = {k: z[k] for k in ("idx_g", "idx_s", "idx_p")}
        plotting = {"limits": np.array([0, 640, -400, 0])}
        super().__init__(W, coords=z["coords"], plotting=plotting, **kwargs)


class Ring(Graph):
    r"""Ring graph: vertex i is linked to i +- 1..k (pygsp/graphs/ring.py)."""

    def __init__(self, N=64, k=1, **kwargs):
        if N < 3:
            raise ValueError("There should be at least 3 vertices.")
        if 2 * k > N:
            raise ValueError("Too many neighbors requested.")
        self.k = k
        rows, cols = [], []
        idx = np.arange(N)
        for s in range(1, k + 1):
            rows.append(idx)
            cols.append((idx + s) % N)
        rows, cols = np.concatenate(rows), np.concatenate(cols)
        W = sparse.coo_matrix((np.ones(rows.size), (rows, cols)), shape=(N, N)).tocsr()
        W = W + W.T
        W.data[:] = 1.0                             # unit weights (antipodal edge met twice)
        theta = 2 * np.pi * idx / N
        super().__init__(W, coords=np.stack([np.cos(theta), np.sin(theta)], axis=1), **kwargs)


class Grid2d(Graph):
    r"""N1 x N2 grid with 4-neighbour (5-point stencil) connectivity, unit weights.

    Same graph and row-major vertex numbering as pygsp/graphs/grid2d.py:40-89.
    """

    def __init__(self, N1=16, N2=None, backend="device", **kwargs):
        if N2 is None:
            N2 = N1
        self.N1, self.N2 = N1, N2
        N = N1 * N2
        if backend == "device":                     # stencil written straight into HBM
            W = grid2d_adjacency_device(N1, N2, kwargs.get("dtype"), kwargs.get("device"))
        else:
            right = np.ones(N - 1)
            right[N2 - 1::N2] = 0                   # no edge across a row end
            W = sparse.diags([right, np.ones(N - N2)], [1, N2], shape=(N, N), format="csr")
            W.eliminate_zeros()
            W = (W + W.T).tocsr()
        x = np.tile(np.arange(N2) / float(N2), N1)
        y = np.repeat(np.arange(N1)[::-1] / float(N1), N2)
        super().__init__(W, coords=np.stack([x, y], axis=1), **kwargs)


def _device_of(device):
    torch = nat.require_cuda()
    return torch.device(device if device is not None else "cuda:%d" % torch.cuda.current_device())


def grid2d_adjacency_device(N1, N2, dtype=None, device=None):
    """Grid2d adjacency built by ``gsp_grid2d_*`` (no host matrix)."""
    torch = nat.require_cuda()
    dev, dt = _device_of(device), _torch_dtype(torch, dtype)
    shape = (nat.i64(N1), nat.i64(N2))
    return DeviceCSR.from_counts(
        (N1 * N2, N1 * N2), dt, dev,
        lambda st, ip, nnz: nat.call("gsp_grid2d_count", *shape, ip, nnz, st),
        lambda st, ip, ix, d: nat.call("gsp_grid2d_fill_" + nat.suffix(dt), *shape, ip, ix, d, st),
        "graph")


def _device_points(points, dev):
    torch = nat.require_cuda()
    return torch.as_tensor(np.asarray(points, dtype=np.float64) if not torch.is_tensor(points)
                           else points).to(device=dev, dtype=torch.float64).contiguous()


def _check_order(p):
    p = float(p)
    if not p >= 1:
        raise ValueError("Only p-norms with 1<=p<=infinity permitted (p = {}).".format(p))
    return p


def _require_finite(pts):
    """``ValueError`` unless every coordinate is finite, as cKDTree: a NaN or an infinity has
    no place in a distance order."""
    torch = nat.require_cuda()
    if not bool(torch.isfinite(pts).all()):
        raise ValueError("data must be finite")


# gsp_knn_grid's bounds: cells per axis (so that ring indices stay in int32) and cells per point
# (so that the cell table stays a few entries per point)
_GRID_AXIS_CELLS = 2 ** 30
_GRID_CELLS_PER_POINT = 4


def _knn_grid_cells(lo, hi, n, points_per_cell):
    """Cells per axis of the uniform grid that ``gsp_knn_grid`` lays over the box [lo, hi] of
    n points.

    Cubic cells of side h hold ``points_per_cell`` points on average: h^m = volume *
    points_per_cell / n over the m axes whose span reaches h.  An axis thinner than one cell (a
    line, a plane, all points equal, a spread at rounding level) gets one cell and leaves the
    volume, so that it cannot shrink the cells of the others; h is recomputed until no axis drops
    out.  Counts are clipped in float64 before the integer cast: every axis gets 1 .. 2^30 cells,
    all of them together at most 4 n.
    """
    with np.errstate(over="ignore"):
        span = np.asarray(hi, dtype=np.float64) - np.asarray(lo, dtype=np.float64)
    if not np.isfinite(span).all():
        raise ValueError("the range of the coordinates must be finite")
    if not points_per_cell > 0:
        raise ValueError("points_per_cell must be positive")
    cells = np.ones(span.shape)
    live = span > 0
    while live.any():
        # in logarithms: the volume of a thin box can underflow
        h = np.exp((np.log(span[live]).sum() + np.log(points_per_cell / n)) / live.sum())
        thin = live & (span < h)
        if not thin.any():
            cells[live] = np.minimum(np.floor(span[live] / h), _GRID_AXIS_CELLS)
            break
        live &= ~thin
    cells = cells.astype(np.int64)
    while math.prod(cells.tolist()) > min(_GRID_CELLS_PER_POINT * n, 2 ** 31 - 1):
        cells = np.maximum(cells // 2, 1)
    return cells.astype(np.int32)


def knn_device(points, k, device=None, points_per_cell=3.0, p=2):
    """k nearest neighbours of every point (self excluded by index) on the GPU.

    Stands in for ``scipy.spatial.KDTree(X).query(X, k + 1, p=p)`` (nngraph.py:213-216):
    returns (nn, dist), both (N, k) CUDA tensors, ascending (distance, id); k <= 32.  Euclidean
    2-D / 3-D clouds are searched on a cell grid (``gsp_knn_grid``), every other dimension and
    Minkowski order p >= 1 (inf included) exhaustively (``gsp_knn_brute``); both are exact and
    give the same lists, bit for bit.  The grid's cells hold ``points_per_cell`` points on average
    (:func:`_knn_grid_cells`).  ``ValueError`` for a coordinate that is not finite, as cKDTree.
    """
    torch = nat.require_cuda()
    dev = _device_of(device)
    p = _check_order(p)
    pts = _device_points(points, dev)
    n, dim = pts.shape
    if p != 2 or dim not in (2, 3):
        _require_finite(pts)
        nn = torch.empty((n, k), dtype=torch.int32, device=dev)
        dist = torch.empty((n, k), dtype=torch.float64, device=dev)
        with torch.cuda.device(dev):
            nat.call("gsp_knn_brute", nat.i64(n), nat.i32(dim), pts, nat.i32(k), nat.f64(p), nn,
                     dist, nat.stream_ptr(dev))
        return nn, dist
    # min and max propagate NaN, so a coordinate that is not finite reaches lo or hi, and
    # _knn_grid_cells refuses the box
    lo = pts.min(dim=0).values.cpu().numpy().astype(np.float64)
    hi = pts.max(dim=0).values.cpu().numpy().astype(np.float64)
    cells = _knn_grid_cells(lo, hi, n, points_per_cell)
    nn = torch.empty((n, k), dtype=torch.int32, device=dev)
    dist = torch.empty((n, k), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        nat.call("gsp_knn_grid", nat.i64(n), nat.i32(dim), pts, nat.i32(k),
                 np.ascontiguousarray(lo), np.ascontiguousarray(hi), np.ascontiguousarray(cells),
                 nn, dist, nat.stream_ptr(dev))
    return nn, dist


def knn_adjacency_device(points, k, sigma=None, dtype=None, device=None):
    """Symmetric Gaussian k-NN adjacency (nngraph.py:213-226,289-297) built on the GPU."""
    torch = nat.require_cuda()
    dev, dt = _device_of(device), _torch_dtype(torch, dtype)
    nn, dist = knn_device(points, k, dev)
    if sigma is None:
        sigma = float(dist.mean().item())
    return _knn_gauss_csr(nn, dist, sigma, dt).symmetrize("average"), sigma


def _knn_gauss_csr(nn, dist, sigma, dt):
    """Directed Gaussian k-NN matrix W[i, nn[i]] = exp(-dist[i]^2 / sigma) of (n, k) neighbour
    lists, sorted rows, in dtype dt on the lists' device (``gsp_knn_to_csr_*``)."""
    torch = nat.require_cuda()
    (n, k), dev = nn.shape, nn.device
    indptr = torch.empty(n + 1, dtype=torch.int32, device=dev)
    indices = torch.empty(n * k, dtype=torch.int32, device=dev)
    data = torch.empty(n * k, dtype=dt, device=dev)
    with torch.cuda.device(dev):
        nat.call("gsp_knn_to_csr_" + nat.suffix(dt), nat.i64(n), nat.i32(k), nn, dist,
                 nat.f64(sigma), indptr, indices, data, nat.stream_ptr(dev))
    return DeviceCSR(indptr, indices, data, (n, n))


def radius_device(points, epsilon, p=2, device=None):
    """Radius neighbourhoods of every point on the GPU: a (N, N) DeviceCSR of float64 distances.

    Row i holds the j != i with ``dist(x_i, x_j) <= epsilon`` in the Minkowski metric of order p,
    sorted by column -- ``KDTree(X).query_ball_point(X, r=epsilon, p=p)`` and the self filter of
    nngraph.py:228-283.  The number of entries is read once; ``ValueError`` when it does not fit
    int32 CSR offsets or the free device memory, before anything is allocated for them, and for a
    coordinate that is not finite.
    """
    torch = nat.require_cuda()
    dev = _device_of(device)
    p = _check_order(p)
    pts = _device_points(points, dev)
    _require_finite(pts)
    n, dim = pts.shape
    cloud = (nat.i64(n), nat.i32(dim), pts, nat.f64(epsilon), nat.f64(p))

    def fits_in_memory(nnz):
        free = torch.cuda.mem_get_info(dev)[0]
        if 12 * nnz > free:
            raise ValueError("the radius graph has %d entries (%d bytes): more than the free "
                             "device memory (%d bytes)" % (nnz, 12 * nnz, free))
    return DeviceCSR.from_counts(
        (n, n), torch.float64, dev,
        lambda st, ip, nnz: nat.call("gsp_radius_count", *cloud, ip, nnz, st),
        lambda st, ip, ix, d: nat.call("gsp_radius_fill_f64", *cloud, ip, ix, d, st),
        "radius graph", check=fits_in_memory)


def _gauss_weights_device(D, sigma, dt):
    """DeviceCSR of exp(-d^2 / sigma) on the structure of a distance matrix D."""
    torch = nat.require_cuda()
    w = torch.empty(D.nnz, dtype=dt, device=D.device)
    with torch.cuda.device(D.device):
        nat.call("gsp_gauss_weights_" + nat.suffix(dt), nat.i64(D.nnz), D.data, nat.f64(sigma), w,
                 nat.stream_ptr(D.device))
    return DeviceCSR(D.indptr, D.indices, w, D.shape)


_DIST_ORDER = {"euclidean": 2.0, "manhattan": 1.0, "max_dist": np.inf}
_SYMMETRIZE_TYPES = ("average", "maximum", "fill", "tril", "triu")
_logger = utils.build_logger(__name__)


def _minkowski_order(dist_type, order, use_flann):
    """(p, renumbering) from NNGraph's dist_type and order.

    ``order`` renumbers vertices (None, 'morton' or a permutation).  The reference uses it as
    the Minkowski order instead (nngraph.py:162-167); a real scalar was never a renumbering, so
    with dist_type='minkowski' a scalar is p.  Without one p is the reference's default 0, which
    its scikit-learn branch (use_flann=True) turns into the Euclidean metric and KDTree refuses.
    """
    if dist_type not in ("euclidean", "manhattan", "max_dist", "minkowski"):
        raise ValueError("Unknown dist_type {}.".format(dist_type))
    if dist_type != "minkowski":
        return _DIST_ORDER[dist_type], order
    scalar = order is not None and np.ndim(order) == 0 and not isinstance(order, str)
    p = float(order) if scalar else 0.0
    if p <= 0 and use_flann:
        p = 2.0
    return _check_order(p), (None if scalar else order)


def _host_knn(X, k, p):
    D, NN = spatial.cKDTree(X).query(X, k=k + 1, p=p, workers=-1)
    return D[:, 1:], NN[:, 1:]


def _host_radius(X, epsilon, p):
    """Rows of query_ball_point without self (sorted) and their distances, as COO arrays."""
    lists = spatial.cKDTree(X).query_ball_point(X, r=epsilon, p=p, workers=-1,
                                                return_sorted=True)
    rows = np.repeat(np.arange(X.shape[0]), [len(nb) for nb in lists])
    cols = np.concatenate([np.asarray(nb, dtype=np.int64) for nb in lists]) if len(lists) else \
        np.zeros(0, dtype=np.int64)
    keep = rows != cols
    rows, cols = rows[keep], cols[keep]
    diff = np.abs(X[rows] - X[cols])
    if p == 2:
        dist = np.sqrt(np.sum(diff * diff, axis=1))
    elif p == 1:
        dist = np.sum(diff, axis=1)
    elif np.isinf(p):
        dist = diff.max(axis=1) if diff.size else np.zeros(0)
    else:
        dist = np.sum(diff ** p, axis=1) ** (1.0 / p)
    return rows, cols, dist


class NNGraph(Graph):
    r"""Nearest-neighbour graph of a point cloud with Gaussian weights.

    pygsp/graphs/nngraphs/nngraph.py:92-299 with its ``center`` / ``rescale`` preprocessing
    (:127-136).  ``NNtype='knn'``: the k nearest neighbours j of every i, sigma = mean of the
    k neighbour distances; ``NNtype='radius'``: every j != i within ``epsilon``, sigma = mean of
    those distances (``ValueError`` when there is none).  ``w_ij = exp(-d_ij^2 / sigma)`` for
    every metric, then ``utils.symmetrize(W, symmetrize_type)``.  ``dist_type``: 'euclidean',
    'manhattan', 'max_dist' or 'minkowski' (order p >= 1 given as ``order``, see
    :func:`_minkowski_order`).  The search is always exact: ``use_flann`` is accepted and
    changes nothing.

    ``backend=None`` picks the device for k <= 32 (a cell grid for Euclidean k-NN of 2-D / 3-D
    clouds, an exhaustive search otherwise; csrc/generate.cu, csrc/neighbors.cu) and scipy's
    cKDTree on the host for larger k; ``'device'`` / ``'host'`` force the choice.  ``Xin`` may
    be a CUDA tensor (the patch graphs build their features on the device).
    """

    def __init__(self, Xin, k=10, sigma=None, center=True, rescale=True, order=None,
                 backend=None, *, NNtype="knn", use_flann=False, epsilon=0.01,
                 symmetrize_type="average", dist_type="euclidean", **kwargs):
        if NNtype not in ("knn", "radius"):
            raise ValueError("Unknown NNtype {}".format(NNtype))
        if symmetrize_type not in _SYMMETRIZE_TYPES:
            raise ValueError("Unknown symmetrization method {}.".format(symmetrize_type))
        p, order = _minkowski_order(dist_type, order, use_flann)
        if use_flann:
            _logger.debug("use_flann: the neighbour search is exact, FLANN is not used")
        self.NNtype, self.use_flann, self.epsilon = NNtype, use_flann, epsilon
        self.symmetrize_type, self.dist_type = symmetrize_type, dist_type
        self.center, self.rescale = center, rescale
        on_device = _is_tensor(Xin)
        if not on_device:
            Xin = np.asarray(Xin, dtype=np.float64)
        self.Xin = Xin
        N, d = Xin.shape
        if k >= N:
            raise ValueError("The number of neighbors (k={}) must be smaller than the number "
                             "of nodes ({}).".format(k, N))
        if on_device:
            torch = nat.require_cuda()
            X = Xin.to(torch.float64)
            X = X - X.mean(dim=0) if center else X.clone()
            if rescale:
                span = X.max(dim=0).values - X.min(dim=0).values
                radius = 0.5 * float(torch.linalg.vector_norm(span, 2).item())
                X *= (np.power(N, 1.0 / float(min(d, 3))) / 10.0) / radius
        else:
            X = Xin - Xin.mean(axis=0) if center else Xin.copy()
            if rescale:
                radius = 0.5 * np.linalg.norm(X.max(axis=0) - X.min(axis=0), 2)
                X *= (np.power(N, 1.0 / float(min(d, 3))) / 10.0) / radius
        if order is not None:
            if on_device:
                X = X[morton_order_device(X) if order == "morton"
                      else torch.as_tensor(np.asarray(order), device=X.device).long()]
            else:
                X = X[morton_order(X) if order == "morton" else np.asarray(order)]
        if backend is None:     # the device searches cover k <= 32
            backend = "device" if k <= 32 else "host"
        self.k = k
        if backend == "device":
            W, sigma = self._device_adjacency(X, k, sigma, p, epsilon, kwargs.get("dtype"),
                                              kwargs.get("device"))
        else:
            W, sigma = self._host_adjacency(X.cpu().numpy() if on_device else X, k, sigma, p,
                                            epsilon)
        self.sigma = sigma
        super().__init__(W, coords=X.cpu().numpy() if on_device else X, **kwargs)

    def _device_adjacency(self, X, k, sigma, p, epsilon, dtype, device):
        torch = nat.require_cuda()
        dev, dt = _device_of(device), _torch_dtype(torch, dtype)
        if self.NNtype == "knn":     # with 'average': the steps of knn_adjacency_device
            nn, dist = knn_device(X, k, dev, p=p)
            if sigma is None:
                sigma = float(dist.mean().item())
            W = _knn_gauss_csr(nn, dist, sigma, dt)
        else:
            D = radius_device(X, epsilon, p, dev)
            if sigma is None:
                if D.nnz == 0:
                    raise ValueError("No neighbors found")
                sigma = float(D.data.mean().item())
            W = _gauss_weights_device(D, sigma, dt)
        return W.symmetrize(self.symmetrize_type), sigma

    def _host_adjacency(self, X, k, sigma, p, epsilon):
        N = X.shape[0]
        if self.NNtype == "knn":
            D, NN = _host_knn(X, k, p)
            if sigma is None:
                sigma = np.mean(D)
            rows, cols, dist = np.repeat(np.arange(N), k), NN.ravel(), D.ravel()
        else:
            rows, cols, dist = _host_radius(X, epsilon, p)
            if sigma is None:
                if dist.size == 0:
                    raise ValueError("No neighbors found")
                sigma = np.mean(dist)
        W = sparse.csr_matrix((np.exp(-dist ** 2 / float(sigma)), (rows, cols)), shape=(N, N))
        return utils.symmetrize(W, self.symmetrize_type).tocsr(), sigma


def _is_tensor(x):
    return type(x).__module__.startswith("torch") and hasattr(x, "data_ptr")


def _patch_pad_index(size, lo, hi):
    """Source index of every position of np.pad(mode='symmetric') along one axis."""
    i = np.arange(-lo, size + hi)
    period = 2 * size
    i = np.mod(i, period)
    return np.where(i < size, i, period - 1 - i)


def image_patches_device(img, patch_shape=(3, 3), device=None):
    """Patch features of ImgPatches (imgpatches.py:51-105) as an (h*w, r*c*C) float64 CUDA
    tensor: np.pad(img, mode='symmetric') with the reference's pad widths, then one row per
    pixel in row-major order holding the r x c window (x C channels, channel fastest) --
    skimage's view_as_windows + reshape, done by gather and unfold on the device."""
    torch = nat.require_cuda()
    dev = _device_of(device)
    im = _device_points(img, dev) if not _is_tensor(img) else img.to(dev, torch.float64)
    if im.dim() == 2:
        im = im[:, :, None]
    elif im.dim() != 3:
        raise ValueError("Image should be a 2D (gray) or 3D (h, w, C) array.")
    h, w, ch = im.shape
    r, c = (patch_shape[0], patch_shape[1]) if len(patch_shape) > 1 else \
        (patch_shape[0], patch_shape[0])
    rows = _patch_pad_index(h, int((r - 0.5) / 2.0), int((r + 0.5) / 2.0))
    cols = _patch_pad_index(w, int((c - 0.5) / 2.0), int((c + 0.5) / 2.0))
    padded = im[torch.from_numpy(rows).to(dev)][:, torch.from_numpy(cols).to(dev)]
    win = padded.unfold(0, r, 1).unfold(1, c, 1)          # (h, w, C, r, c)
    return win.permute(0, 1, 3, 4, 2).reshape(h * w, r * c * ch).contiguous()


class ImgPatches(NNGraph):
    r"""Nearest-neighbour graph between the patches of an image (imgpatches.py:51-105).

    Every pixel's feature vector is the ``patch_shape`` window centred on it (symmetric padding
    at the borders), all channels stacked: ``r * c * C`` values for an (h, w, C) image, ``r * c``
    for a gray one.  The features are built on the device (:func:`image_patches_device`) and
    kept in ``Xin``; keyword arguments go to :class:`NNGraph`.
    """

    def __init__(self, img, patch_shape=(3, 3), **kwargs):
        self.img = img
        self.patch_shape = patch_shape
        patches = image_patches_device(img, patch_shape, kwargs.get("device"))
        super().__init__(patches, **kwargs)


class Grid2dImgPatches(Graph):
    r"""Union of a patch graph and the image's 2-D grid graph (grid2dimgpatches.py:37-43).

    ``W = aggregate(Wp, Wg)`` of the :class:`ImgPatches` adjacency Wp and the
    :class:`Grid2d` adjacency Wg.  The default ``Wp + Wg`` is summed on the device (COO
    concatenation, then ``DeviceCSR.from_coo``, which adds duplicates); a user-supplied
    ``aggregate`` receives both as SciPy CSR matrices, as in the reference.  Keyword arguments
    go to :class:`ImgPatches`; the graph takes the grid's coordinates.
    """

    def __init__(self, img, aggregate=None, **kwargs):
        torch = nat.require_cuda()
        h, w = img.shape[0], img.shape[1]
        dt, dev = kwargs.get("dtype"), kwargs.get("device")
        self.Gg = Grid2d(h, w, dtype=dt, device=dev)
        self.Gp = ImgPatches(img, **kwargs)
        if aggregate is None:
            Wp, Wg = self.Gp.W, self.Gg.W
            W = DeviceCSR.from_coo(torch.cat([row_ids(Wp.indptr), row_ids(Wg.indptr)]),
                                   torch.cat([Wp.indices, Wg.indices]),
                                   torch.cat([Wp.data, Wg.data.to(Wp.dtype)]), (h * w, h * w))
        else:
            W = aggregate(self.Gp.W.to_scipy(), self.Gg.W.to_scipy())
        super().__init__(W, coords=self.Gg.coords, plotting=self.Gg.plotting,
                         dtype=dt, device=dev)


class Sensor(NNGraph):
    r"""Random sensor network: N uniform points in the unit square, k-NN graph.

    pygsp/graphs/nngraphs/sensor.py:50-75 (non-distributed variant):
    ``coords = default_rng(seed).uniform(0, 1, (N, 2))``, ``NNGraph(k=k,
    rescale=False, center=False)``.  ``order='morton'`` renumbers the vertices
    along a Z-curve (an isomorphic graph with gather-friendly numbering).
    """

    def __init__(self, N=64, k=6, seed=None, order=None, backend=None, **kwargs):
        self.seed = seed
        kwargs["backend"] = backend
        coords = np.random.default_rng(seed).uniform(0, 1, (N, 2))
        kwargs.setdefault("plotting", {"limits": np.array([0, 1, 0, 1])})
        super().__init__(coords, k=k, center=False, rescale=False, order=order, **kwargs)


class SensorStrips:
    r"""Row block of a Sensor-type k-NN graph on the strip domain [0, P) x [0, 1).

    Weak-scaling input of the partitioned path: strip q holds ``n_per`` uniform
    points (``default_rng(seed + q)``, Morton-numbered inside the strip, global ids
    q*n_per ...), every strip is one rank's row block.  A rank regenerates its two
    neighbour strips, so no point data crosses ranks; the graph is exactly the k-NN
    graph of the union of all strips with NNGraph's weights and 'average'
    symmetrisation (nngraph.py:218-226,289-297), as ``tests`` check against a
    directly built global graph.  Host-side input fabrication (scipy cKDTree).
    """

    def __init__(self, rank, parts, n_per, k=10, seed=0):
        self.rank, self.parts, self.n_per, self.k = rank, parts, n_per, k
        self.strips = [q for q in (rank - 1, rank, rank + 1) if 0 <= q < parts]
        pts = []
        for q in self.strips:
            p = np.random.default_rng(seed + q).uniform(0, 1, (n_per, 2))
            p = p[morton_order(p)]
            p[:, 0] += q
            pts.append(p)
        self.points = np.concatenate(pts)
        self.own_lo = self.strips.index(rank) * n_per
        own = np.arange(self.own_lo, self.own_lo + n_per)
        margin = 8.0 * np.sqrt(k / (np.pi * n_per))
        x = self.points[:, 0]
        near = (np.abs(x - rank) < margin) | (np.abs(x - (rank + 1)) < margin)
        near[own] = False
        self.sel = np.concatenate([own, np.flatnonzero(near)])
        tree = spatial.cKDTree(self.points)
        self.D, self.NN = tree.query(self.points[self.sel], k=k + 1, workers=-1)
        if self.D[:, -1].max() * 2 >= margin:
            raise RuntimeError("strip margin too small for this density")
        self.coords = self.points[own]

    def distance_sum(self):
        """(sum, count) of the own points' neighbour distances: sigma = global mean."""
        d = self.D[:self.n_per, 1:]
        return float(d.sum()), int(d.size)

    def adjacency_rows(self, sigma):
        """W[rows of this rank, :] as CSR with GLOBAL column ids."""
        m, k = self.points.shape[0], self.k
        src = np.repeat(self.sel, k)
        A = sparse.csr_matrix((np.exp(-self.D[:, 1:].ravel() ** 2 / float(sigma)),
                               (src, self.NN[:, 1:].ravel())), shape=(m, m))
        S = ((A + A.T) / 2).tocsr()[self.own_lo:self.own_lo + self.n_per]
        S.sort_indices()
        local = S.indices.astype(np.int64)
        strip = np.asarray(self.strips, dtype=np.int64)[local // self.n_per]
        gcol = strip * self.n_per + local % self.n_per
        n_global = self.parts * self.n_per
        # global ids keep the local order inside a strip and strips are ascending,
        # so the columns stay sorted
        return sparse.csr_matrix((S.data, gcol, S.indptr), shape=(self.n_per, n_global))


def morton_order_device(coords, bits=None):
    """:func:`morton_order` on the GPU: the same integer codes (float64 quantisation, bit
    interleave) and a stable sort, so the permutation is identical to the host one."""
    torch = nat.require_cuda()
    n, d = coords.shape
    if bits is None:
        bits = 21 if d <= 3 else 64 // d
    c = coords.to(torch.float64)
    lo = c.min(dim=0).values
    span = torch.clamp(c.max(dim=0).values - lo, min=1e-300)
    q = torch.clamp(((c - lo) / span * float(1 << bits)).to(torch.int64), max=(1 << bits) - 1)
    code = torch.zeros(n, dtype=torch.int64, device=coords.device)
    for b in range(bits):
        for k in range(d):
            code |= ((q[:, k] >> b) & 1) << (b * d + k)
    return torch.sort(code, stable=True).indices


def _unit_ball(dim):
    return {2: np.pi, 3: 4.0 * np.pi / 3.0}[dim]


class KnnSlabs:
    r"""Row block of ONE k-NN graph of ``parts * n_per`` points in the unit square / cube.

    Input of the partitioned path for BASELINE configs[4] (synthetic k-NN point cloud, k = 16,
    3-D, 5e7 points on 8 GPUs) and, in 2-D, the strong-scaling twin of ``Sensor``.  Slab q =
    ``{x_0 in [q/P, (q+1)/P)}`` holds ``n_per`` uniform points (``default_rng(seed + q)``,
    Morton-numbered inside the slab, global ids ``q * n_per ...``) and is rank q's row block.
    A rank regenerates its two neighbour slabs and keeps their points within ``2 m`` of its
    faces, searches the k nearest neighbours of every kept point on the GPU (``gsp_knn_grid``)
    and uses the lists of its own points and of the neighbour points within ``m`` (their
    search balls lie inside the kept set when every k-th distance is <= m, which is checked).
    Weights, sigma = global mean neighbour distance and the 'average' symmetrisation are
    NNGraph's (pygsp/graphs/nngraphs/nngraph.py:213-226,289-297); the result is exactly the row
    block of the graph of the union of all slabs (tests compare with ``NNGraph``).
    ``backend='host'`` runs the same plan with scipy's cKDTree (CPU tests of the host logic).
    """

    def __init__(self, rank, parts, n_per, dim=3, k=16, seed=0, backend="device",
                 margin_factor=2.5, device=None):
        self.rank, self.parts, self.n_per, self.dim, self.k = rank, parts, n_per, dim, k
        self.backend = backend
        n_global = parts * n_per
        self.n_global = n_global
        r_mean = (k / (_unit_ball(dim) * n_global)) ** (1.0 / dim)
        self.margin = m = margin_factor * r_mean
        if parts > 1 and 2 * m > 1.0 / parts:
            raise ValueError("slabs thinner than the search margin: fewer parts or more points")
        strips = [q for q in (rank - 1, rank, rank + 1) if 0 <= q < parts]
        x_lo, x_hi = rank / parts, (rank + 1) / parts
        pts, gid, near = [], [], []
        for q in strips:
            p = np.random.default_rng(seed + q).uniform(0, 1, (n_per, dim))
            p[:, 0] = (p[:, 0] + q) / parts
            if backend == "device":
                torch = nat.require_cuda()
                dev = _device_of(device)
                pt = torch.from_numpy(p).to(dev)
                pt = pt[morton_order_device(pt)]
                ids = torch.arange(q * n_per, (q + 1) * n_per, device=dev)
                if q != rank:
                    dist = (x_lo - pt[:, 0]) if q < rank else (pt[:, 0] - x_hi)
                    keep = dist < 2 * m
                    pt, ids, dist = pt[keep], ids[keep], dist[keep]
                    near.append(dist < m)
                else:
                    near.append(torch.ones(n_per, dtype=torch.bool, device=dev))
                    self.own_lo = int(sum(x.shape[0] for x in pts))
            else:
                p = p[morton_order(p)]
                ids = np.arange(q * n_per, (q + 1) * n_per)
                if q != rank:
                    dist = (x_lo - p[:, 0]) if q < rank else (p[:, 0] - x_hi)
                    keep = dist < 2 * m
                    p, ids, dist = p[keep], ids[keep], dist[keep]
                    near.append(dist < m)
                else:
                    near.append(np.ones(n_per, dtype=bool))
                    self.own_lo = int(sum(x.shape[0] for x in pts))
                pt = p
            pts.append(pt)
            gid.append(ids)
        if backend == "device":
            torch = nat.require_cuda()
            self.points = torch.cat(pts)
            self.gid = torch.cat(gid)
            self.used = torch.cat(near)
            self.coords = self.points[self.own_lo:self.own_lo + n_per]
            self.NN, self.D = knn_device(self.points, k, self.points.device)
            kth = float(self.D[self.used, -1].max().item())
        else:
            self.points = np.concatenate(pts)
            self.gid = np.concatenate(gid)
            self.used = np.concatenate(near)
            self.coords = self.points[self.own_lo:self.own_lo + n_per]
            D, NN = spatial.cKDTree(self.points).query(self.points, k=k + 1, workers=-1)
            self.D, self.NN = D[:, 1:], NN[:, 1:]
            kth = float(self.D[self.used, -1].max())
        if parts > 1 and kth > m:
            raise RuntimeError("search margin too small for this density (k-th distance %g > %g): "
                               "raise margin_factor" % (kth, m))

    def distance_sum(self):
        """(sum, count) of the own points' neighbour distances: sigma = global mean."""
        d = self.D[self.own_lo:self.own_lo + self.n_per]
        if self.backend == "device":
            return float(d.sum(dtype=d.dtype).item()), int(d.numel())
        return float(d.sum()), int(d.size)

    def adjacency_rows(self, sigma):
        """W[rows of this rank, :] as a host CSR with GLOBAL column ids (host backend)."""
        m, k = self.points.shape[0], self.k
        D, NN, used = self.D, self.NN, self.used
        if self.backend == "device":
            D, NN, used = D.cpu().numpy(), NN.cpu().numpy().astype(np.int64), used.cpu().numpy()
        gid = self.gid if self.backend != "device" else self.gid.cpu().numpy()
        src = np.repeat(np.flatnonzero(used), k)
        A = sparse.csr_matrix((np.exp(-D[used].ravel() ** 2 / float(sigma)),
                               (src, NN[used].ravel())), shape=(m, m))
        S = ((A + A.T) / 2).tocsr()[self.own_lo:self.own_lo + self.n_per]
        S.sort_indices()
        # kept points are in ascending global order, so renaming keeps the rows sorted
        return sparse.csr_matrix((S.data, gid[S.indices], S.indptr),
                                 shape=(self.n_per, self.n_global))

    def laplacian_rows_device(self, sigma, dtype=None):
        """Rows of L = D - W of this rank, built in HBM: (indptr int32, indices int32 GLOBAL
        ids, data) tensors in canonical CSR order (sorted rows, diagonal in place), and dw."""
        torch = nat.require_cuda()
        if self.backend != "device":
            raise ValueError("laplacian_rows_device needs backend='device'")
        dev, dt = self.points.device, _torch_dtype(torch, dtype)
        n = self.n_per
        # unused rows (kept points farther than `margin` from the slab) get zero-weight lists:
        # an infinite distance gives exp(-inf) = 0 and the zeros are dropped below
        dist = torch.where(self.used[:, None], self.D, torch.full_like(self.D, float("inf")))
        W = _knn_gauss_csr(self.NN, dist, sigma, dt).symmetrize("average")
        del dist
        ptr = W.indptr[self.own_lo:self.own_lo + n + 1]
        a, b = int(ptr[0].item()), int(ptr[-1].item())
        cols, vals = W.indices[a:b].long(), W.data[a:b]
        rows = row_ids(ptr)
        keep = vals != 0
        rows, vals = rows[keep], vals[keep]
        gcol = self.gid[cols[keep]]
        del cols, keep, W
        counts = torch.bincount(rows, minlength=n)
        dw = torch.segment_reduce(vals.double(), "sum", lengths=counts)
        # L row i = -W row i with dw_i inserted at the diagonal's sorted position
        gdiag = self.gid[self.own_lo:self.own_lo + n]
        before = gcol < gdiag[rows]
        n_before = torch.segment_reduce(before.double(), "sum", lengths=counts).long()
        has_diag = dw != 0                                  # isolated vertex: empty row (graph.py:620)
        l_counts = counts + has_diag.long()
        l_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(l_counts, 0, out=l_ptr[1:])
        nnz = int(l_ptr[-1].item())
        if nnz >= 2 ** 31:
            raise ValueError("the rank's rows of L must fit int32 offsets (nnz = %d)" % nnz)
        w_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        torch.cumsum(counts, 0, out=w_ptr[1:])
        pos = torch.arange(rows.numel(), device=dev) - w_ptr[rows] + l_ptr[rows] + \
            (~before & has_diag[rows]).long()
        l_idx = torch.empty(nnz, dtype=torch.int32, device=dev)
        l_val = torch.empty(nnz, dtype=dt, device=dev)
        l_idx[pos] = gcol.int()
        l_val[pos] = -vals
        dpos = (l_ptr[:-1] + n_before)[has_diag]
        l_idx[dpos] = gdiag[has_diag].int()
        l_val[dpos] = dw[has_diag].to(dt)
        return l_ptr.int(), l_idx, l_val, dw


def laplacian_rows(W_rows, row_offset):
    """Rows of the combinatorial Laplacian D - W from rows of a SYMMETRIC adjacency.

    Host helper of the partitioned path: dw of a row block is its row sums, so the
    rows of L are built without the rest of the matrix (graph.py:618-620)."""
    W_rows = W_rows.tocsr()
    n_local, n = W_rows.shape
    dw = np.asarray(W_rows.sum(axis=1)).ravel()
    D = sparse.csr_matrix((dw, (np.arange(n_local), np.arange(n_local) + row_offset)),
                          shape=(n_local, n))
    L = (D - W_rows).tocsr()
    L.eliminate_zeros()
    L.sort_indices()
    return L, dw


def sbm_adjacency(N=1024, k=5, z=None, p=0.7, q=None, seed=None):
    r"""Adjacency of an undirected, loop-free stochastic block model, vectorised.

    Same model as pygsp/graphs/stochasticblockmodel.py:61-144 with its defaults
    (``z = sort(rng.integers(0, k, N))``, edge (i, j), i != j, present with probability
    ``M[z_i, z_j]``, ``M`` = ``q`` off the diagonal and ``p`` on it, unit weights).  The
    reference draws one uniform per vertex pair in a Python loop (N^2 iterations: unusable
    beyond N ~ 3e3); here every block pair draws its edge COUNT from the binomial law and then
    that many distinct pairs uniformly -- the same distribution, O(edges) work.  The
    random stream necessarily differs from the reference's, so parity is statistical
    (tests/test_generators_cpu.py).
    """
    rng = np.random.default_rng(seed)
    z, M = _sbm_blocks(rng, N, k, z, p, q)
    return _sbm_draw(rng, N, k, z, M), z


def _sbm_blocks(rng, N, k, z, p, q, M=None, sorted_z=True):
    """Block assignment z (drawn from rng when None) and the k x k probability matrix M (built
    from p and q unless given).  ``sorted_z``: the host sampler needs the blocks contiguous."""
    if z is None:
        z = np.sort(rng.integers(0, k, N))
    z = np.asarray(z)
    if M is None:
        pv = np.asarray(p, dtype=np.float64)
        pv = pv * np.ones(k) if pv.size == 1 else pv
        if pv.shape != (k,):
            raise ValueError("Optional parameter p is neither a scalar nor a vector of length k.")
        if q is None:
            q = 0.3 / k
        M = np.asarray(q, dtype=np.float64)
        M = M * np.ones((k, k)) if M.size == 1 else M.copy()
        if M.shape != (k, k):
            raise ValueError("Optional parameter q is neither a scalar nor a matrix of size k x k.")
        M.flat[::k + 1] = pv
    else:
        M = np.array(M, dtype=np.float64)
        if M.shape != (k, k):
            raise ValueError("M must be a matrix of size k x k.")
    if (M < 0).any() or (M > 1).any():
        raise ValueError("Probabilities should be in [0, 1].")
    if z.shape != (N,) or (N and (z.min() < 0 or z.max() >= k)):
        raise ValueError("z must hold N block indices in [0, k).")
    if sorted_z and np.any(np.diff(z) < 0):
        raise ValueError("z must be sorted (blocks contiguous) for the vectorised sampler")
    return z, M


def _sbm_draw(rng, N, k, z, M, directed=False, self_loops=False):
    """One draw of the SBM adjacency (canonical CSR) for blocks z and probabilities M.

    The pair spaces and their decoders are those of the device sampler (graphs/random_graphs.py):
    undirected block pairs b <= a, every ordered pair when directed."""
    from .random_graphs import decode_pairs, pair_space
    start = np.searchsorted(z, np.arange(k), side="left")
    size = np.searchsorted(z, np.arange(k), side="right") - start

    def distinct(n_pairs, m):
        """m distinct integers from range(n_pairs), uniformly."""
        if m == 0:
            return np.zeros(0, dtype=np.int64)
        if m > n_pairs // 3:
            return rng.choice(n_pairs, size=m, replace=False).astype(np.int64)
        got = np.unique(rng.integers(0, n_pairs, int(m * 1.05) + 16))
        while got.size < m:
            got = np.unique(np.concatenate([got, rng.integers(0, n_pairs, m - got.size + 16)]))
        return rng.permutation(got)[:m]

    rows, cols = [], []
    for a in range(k):
        for b in range(k if directed else a + 1):
            kind, n_pairs, width = pair_space(int(size[a]), int(size[b]), a == b, directed,
                                              self_loops)
            if n_pairs == 0 or M[a, b] == 0:
                continue
            idx = distinct(n_pairs, int(rng.binomial(n_pairs, M[a, b])))
            i, j = decode_pairs(kind, idx, width)
            rows.append(start[a] + i)
            cols.append(start[b] + j)
    if rows:
        r = np.concatenate(rows)
        c = np.concatenate(cols)
    else:
        r = c = np.zeros(0, dtype=np.int64)
    if not directed:              # both orientations, a loop once
        off = r != c
        r, c = np.concatenate([r, c[off]]), np.concatenate([c, r[off]])
    W = sparse.coo_matrix((np.ones(r.size), (r, c)), shape=(N, N)).tocsr()
    W.sort_indices()
    return W


class StochasticBlockModel(Graph):
    r"""Stochastic block model graph (pygsp/graphs/stochasticblockmodel.py:61-165).

    Edge (i, j) is present with probability ``M[z_i, z_j]``, unit weights; ``M`` is given or
    built from ``p`` (diagonal) and ``q`` (off the diagonal).  An undirected graph reads the
    lower triangle of ``M``, as the reference does for a sorted ``z``; ``directed`` draws every
    ordered pair, ``self_loops`` the pairs (i, i) too.

    ``backend='host'`` (the default) is :func:`sbm_adjacency`'s sampler: block edge counts from
    the binomial law, then that many distinct pairs; it needs ``z`` sorted.  ``backend='device'``
    walks every block pair's Bernoulli process on the GPU from a Philox key
    (graphs/random_graphs.py); ``z`` need not be sorted there, but an undirected graph with an
    asymmetric ``M`` and an unsorted ``z`` raises ``ValueError``, since a pair's probability
    would then depend on the vertex numbering.  Both draw ``z`` from
    ``np.random.default_rng(seed)``; the device draws one key per trial from it after ``z``.

    ``connected=True`` draws z once and then resamples W until the graph is connected, at most
    ``n_try`` times (None: forever), as stochasticblockmodel.py:125-157 does; it raises the
    reference's ``ValueError`` after ``n_try`` failures.
    """

    def __init__(self, N=1024, k=5, z=None, p=0.7, q=None, seed=None, connected=False,
                 n_try=10, *, M=None, directed=False, self_loops=False, backend="host",
                 **kwargs):
        if backend not in ("host", "device"):
            raise ValueError("Unknown backend {}.".format(backend))
        self.k, self.p, self.q, self.seed = k, p, q, seed
        self.directed, self.self_loops = directed, self_loops
        self.connected, self.n_try = connected, n_try
        rng = np.random.default_rng(seed)
        self.z, self.M = _sbm_blocks(rng, N, k, z, p, q, M, sorted_z=backend == "host")
        if (backend == "device" and not directed and np.any(np.diff(self.z) < 0)
                and not np.array_equal(self.M, self.M.T)):
            raise ValueError("An undirected graph with an asymmetric M needs z sorted: the "
                             "probability of a pair would depend on the vertex numbering.")

        def draw():
            if backend == "host":
                return _sbm_draw(rng, N, k, self.z, self.M, directed, self_loops)
            from .random_graphs import sbm_device
            return sbm_device(N, k, self.z, self.M, directed, self_loops,
                              int(rng.integers(2 ** 63)), kwargs.get("dtype"),
                              kwargs.get("device"))

        W = None
        while n_try is None or n_try > 0:
            W = draw()
            if not connected or Graph(W, dtype=kwargs.get("dtype"),
                                      device=kwargs.get("device")).is_connected():
                break
            if n_try is not None:
                n_try -= 1
        if connected and n_try == 0:
            raise ValueError("The graph could not be connected after {} trials. Increase the "
                             "connection probability or the number of trials.".format(self.n_try))
        if W is None:
            W = draw()
        self.info = {"node_com": self.z, "comm_sizes": np.bincount(self.z, minlength=k),
                     "world_rad": np.sqrt(N)}
        super().__init__(W, **kwargs)

    def _get_extra_repr(self):
        attrs = {"k": self.k}
        if type(self.p) is float:
            attrs["p"] = f"{self.p:.2f}"
        if type(self.q) is float:
            attrs["q"] = f"{self.q:.2f}"
        attrs.update({"directed": self.directed, "self_loops": self.self_loops,
                      "connected": self.connected, "seed": self.seed})
        return attrs
