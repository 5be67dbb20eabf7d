"""Structured graph models and the line graph, built on the device (csrc/structured.cu).

``Path``, ``Comet``, ``Star``, ``Torus``, ``FullConnected``, ``LowStretchTree``, ``RandomRing``
and ``LineGraph`` of pygsp/graphs/{path,comet,star,torus,fullconnected,lowstretchtree,randomring,
linegraph}.py: same signatures, attributes, validation and exceptions, plus the package's
keyword-only ``dtype`` / ``device``.  Each adjacency is written in HBM by the kernels and equals
the reference's bit for bit (float32 data: the float64 values rounded once).  Coordinates are
host NumPy arrays, computed by expressions that give the reference's values exactly.

Kept from the reference on purpose (DESIGN.md section 2): ``LowStretchTree``'s W is directed
and has a self-loop; ``Torus`` adds coinciding neighbours (weight 2, and self-loops for a side
of 1); the line graph of a directed graph has weight 1 between an edge and its reciprocal; a
self-loop edge is a vertex of the line graph with the single entry -1.  The reference's integer
W (``LowStretchTree``, ``LineGraph``) is the engine's float dtype here.
"""
import numpy as np

from .. import _native as nat
from .. import utils
from .csr import DeviceCSR
from .generators import _device_of
from .graph import Graph, _torch_dtype

logger = utils.build_logger(__name__)

_MAX_NNZ = 2 ** 31


def _check_nnz(nnz):
    if nnz >= _MAX_NNZ:
        raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                         "supported.".format(nnz))


def comet_adjacency_device(N, k, directed=False, dtype=None, device=None):
    """Adjacency of ``Comet(N, k)`` (k = 0: ``Path(N, directed)``) by ``gsp_comet_*``."""
    _check_nnz((N - 1) * (1 if directed else 2))
    dt = _torch_dtype(nat.require_cuda(), dtype)
    args = (nat.i64(N), nat.i64(k), nat.i32(directed))
    return DeviceCSR.from_counts(
        (N, N), dt, _device_of(device),
        lambda st, ip, nnz: nat.call("gsp_comet_count", *args, ip, nnz, st),
        lambda st, ip, ix, d: nat.call("gsp_comet_fill_" + nat.suffix(dt), *args, ip, ix, d, st),
        "graph")


class Path(Graph):
    r"""Path graph (pygsp/graphs/path.py): edges i - i+1, or i -> i+1 when ``directed``; unit
    weights, coordinates of ``set_coordinates('line2D')``."""

    def __init__(self, N=16, directed=False, **kwargs):
        if N < 1:
            raise ValueError("negative dimensions are not allowed")
        self.directed = directed
        W = comet_adjacency_device(N, 0, bool(directed), kwargs.get("dtype"), kwargs.get("device"))
        plotting = {"limits": np.array([-1, N, -1, 1])}
        super().__init__(W, plotting=plotting, **kwargs)
        self.set_coordinates("line2D")

    def _get_extra_repr(self):
        return dict(directed=self.directed)


class Comet(Graph):
    r"""Comet graph (pygsp/graphs/comet.py): a star 0 - 1..k and a tail path k - k+1 - ... - N-1.

    The star's branches lie on the unit circle at angles i 2 pi / k, the tail on the x axis at
    abscissae 2, 3, ... from vertex k + 1 on."""

    def __init__(self, N=32, k=12, **kwargs):
        if k > N - 1:
            raise ValueError("The degree of the central vertex k={} must be "
                             "smaller than the number of vertices N={}."
                             "".format(k, N))
        if k < 0:
            raise ValueError("negative dimensions are not allowed")
        self.k = k
        W = comet_adjacency_device(N, k, False, kwargs.get("dtype"), kwargs.get("device"))
        branch = np.arange(k) + 1
        coords = np.zeros((N, 2))
        coords[1:k + 1, 0] = np.cos(branch * 2 * np.pi / k)
        coords[1:k + 1, 1] = np.sin(branch * 2 * np.pi / k)
        coords[k + 1:, 0] = np.arange(2, N - k + 1)
        super().__init__(W, coords=coords, **kwargs)

    def _get_extra_repr(self):
        return dict(k=self.k)


class Star(Comet):
    r"""Star graph (pygsp/graphs/star.py): ``Comet(N, N - 1)``."""

    def __init__(self, N=10, **kwargs):
        plotting = dict(limits=[-1.1, 1.1, -1.1, 1.1])
        plotting.update(kwargs.get("plotting", {}))
        super().__init__(N, N - 1, plotting=plotting, **kwargs)

    def _get_extra_repr(self):
        return dict()


class Torus(Graph):
    r"""Sampled torus (pygsp/graphs/torus.py): Mv rings of Nv vertices, v = i Nv + t linked to
    t +- 1 within its ring and to the same position in rings i +- 1, both modulo.  Coinciding
    neighbours add up, as the reference's duplicate COO entries do."""

    def __init__(self, Nv=16, Mv=None, **kwargs):
        if Mv is None:
            Mv = Nv
        self.Nv, self.Mv = Nv, Mv
        if Nv < 1 or Mv < 1:
            raise ValueError("Nv and Mv must be positive.")
        row0 = {1 % Nv, (Nv - 1) % Nv, (1 % Mv) * Nv, ((Mv - 1) % Mv) * Nv}
        _check_nnz(Nv * Mv * len(row0))          # every row has as many entries as row 0
        dt = _torch_dtype(nat.require_cuda(), kwargs.get("dtype"))
        args = (nat.i64(Nv), nat.i64(Mv))
        W = DeviceCSR.from_counts(
            (Nv * Mv, Nv * Mv), dt, _device_of(kwargs.get("device")),
            lambda st, ip, nnz: nat.call("gsp_torus_count", *args, ip, nnz, st),
            lambda st, ip, ix, d: nat.call("gsp_torus_fill_" + nat.suffix(dt), *args, ip, ix, d,
                                           st),
            "graph")
        phi = np.arange(Mv) * 2 * np.pi / Mv
        theta = np.arange(Nv) * 2 * np.pi / Nv
        radius = 1.5 + np.sin(phi)
        x = np.cos(theta)[None, :] * radius[:, None]     # [i, t]: vertex i Nv + t
        y = np.sin(theta)[None, :] * radius[:, None]
        z = np.broadcast_to(np.cos(phi)[:, None], (Mv, Nv))
        coords = np.stack([x.ravel(), y.ravel(), z.ravel()], axis=1)
        plotting = {"vertex_size": 60, "limits": np.array([-2.5, 2.5, -2.5, 2.5, -2.5, 2.5])}
        super().__init__(W, coords=coords, plotting=plotting, **kwargs)

    def _get_extra_repr(self):
        return dict(Nv=self.Nv, Mv=self.Mv)


class FullConnected(Graph):
    r"""Complete graph (pygsp/graphs/fullconnected.py): every j != i with weight 1.
    ``ValueError`` when N (N - 1) >= 2^31, before anything is allocated."""

    def __init__(self, N=10, **kwargs):
        if N < 0:
            raise ValueError("negative dimensions are not allowed")
        _check_nnz(N * (N - 1))
        dt = _torch_dtype(nat.require_cuda(), kwargs.get("dtype"))
        W = DeviceCSR.from_counts(
            (N, N), dt, _device_of(kwargs.get("device")),
            lambda st, ip, nnz: nat.call("gsp_full_connected_indptr", nat.i64(N), ip, nnz, st),
            lambda st, ip, ix, d: nat.call("gsp_full_connected_fill_" + nat.suffix(dt),
                                           nat.i64(N), ix, d, st),
            "graph")
        plotting = {"limits": np.array([-1, 1, -1, 1])}
        super().__init__(W, plotting=plotting, **kwargs)


def low_stretch_tree_adjacency_device(k, dtype=None, device=None):
    """Adjacency of ``LowStretchTree(k)``: the reference's triplets from
    ``gsp_low_stretch_tree_coo``, assembled by :meth:`DeviceCSR.from_coo`."""
    torch = nat.require_cuda()
    dev, dt = _device_of(device), _torch_dtype(torch, dtype)
    levels = max(int(k), 1)              # k <= 1: the 2 x 2 block alone
    n, nnz = 4 ** levels, 2 * 4 ** levels - 2
    _check_nnz(nnz)
    rows = torch.empty(nnz, dtype=torch.int32, device=dev)
    cols = torch.empty(nnz, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        nat.call("gsp_low_stretch_tree_coo", nat.i32(levels), rows, cols, nat.stream_ptr(dev))
    return DeviceCSR.from_coo(rows, cols, torch.ones(nnz, dtype=dt, device=dev), (n, n))


class LowStretchTree(Graph):
    r"""Root of a low stretch tree on a 2^k x 2^k grid (pygsp/graphs/lowstretchtree.py).

    W is the reference's, directed and with a self-loop at vertex 1 of every 2 x 2 block.
    Vertex v's coordinates: base-4 digit p of v adds 2^p to x when odd and to y when >= 2,
    on top of (1, 1)."""

    def __init__(self, k=6, **kwargs):
        self.k = k
        W = low_stretch_tree_adjacency_device(k, kwargs.get("dtype"), kwargs.get("device"))
        v = np.arange(W.shape[0])
        digits = (v[:, None] // 4 ** np.arange(max(k, 1))) % 4
        step = 2 ** np.arange(max(k, 1))
        coords = np.stack([1 + ((digits & 1) * step).sum(axis=1),
                           1 + ((digits >> 1) * step).sum(axis=1)], axis=1)
        self.root = 4 ** (k - 1)
        plotting = {"edges_width": 1.25, "vertex_size": 75,
                    "limits": np.array([0, 2 ** k + 1, 0, 2 ** k + 1])}
        super().__init__(W, coords=coords, plotting=plotting, **kwargs)

    def _get_extra_repr(self):
        return dict(k=self.k)


class RandomRing(Graph):
    r"""Ring of randomly placed vertices (pygsp/graphs/randomring.py).

    The angles are the reference's: ``np.random.default_rng(seed).uniform(0, 2 pi, N)``,
    sorted, or the given ones, sorted in place.  Edge weights width / (angle difference), with
    width = 2 pi / N, are computed in float64 on the device and rounded once."""

    def __init__(self, N=64, angles=None, seed=None, **kwargs):
        self.seed = seed
        if angles is None:
            rng = np.random.default_rng(seed)
            angles = np.sort(rng.uniform(0, 2 * np.pi, size=N), axis=0)
        else:
            angles = np.asanyarray(angles)
            angles.sort()
            N = len(angles)
            if np.any(angles < 0) or np.any(angles >= 2 * np.pi):
                raise ValueError("Angles should be in [0, 2 pi]")
        self.angles = angles
        if N < 3:
            raise ValueError("There should be at least 3 vertices.")
        _check_nnz(2 * N)
        a = np.asarray(angles, dtype=np.float64)
        gaps = np.append(np.diff(a), 2 * np.pi + a[0] - a[-1])
        width = 2 * np.pi / N
        assert (gaps[gaps != 0].mean() - width) < 1e-10
        torch = nat.require_cuda()
        dev, dt = _device_of(kwargs.get("device")), _torch_dtype(torch, kwargs.get("dtype"))
        a_dev = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        W = DeviceCSR.from_counts(
            (N, N), dt, dev,
            lambda st, ip, nnz: nat.call("gsp_random_ring_count", nat.i64(N), a_dev, ip, nnz, st),
            lambda st, ip, ix, d: nat.call("gsp_random_ring_fill_" + nat.suffix(dt), nat.i64(N),
                                           a_dev, nat.f64(width), ip, ix, d, st),
            "graph")
        coords = np.stack([np.cos(angles), np.sin(angles)], axis=1)
        plotting = {"limits": np.array([-1, 1, -1, 1])}
        super().__init__(W, coords=coords, plotting=plotting, **kwargs)

    def _get_extra_repr(self):
        return dict(seed=self.seed)


def line_graph_adjacency(graph, dtype=None):
    """(adjacency DeviceCSR, sources, targets) of the line graph of ``graph``, on its device.

    Calls ``graph.compute_differential_operator()``.  ``ValueError`` when the line graph would
    hold 2^31 entries or more, raised after the count and before anything else is allocated."""
    dt = _torch_dtype(nat.require_cuda(), graph.dtype if dtype is None else dtype)
    graph.compute_differential_operator()
    D, W, ne = graph.D, graph.W, graph.n_edges
    _, sources, targets, _, _ = graph._edges_device()
    head = (nat.i64(ne), sources, targets, D.indptr)
    tail = (W.indptr, W.indices, nat.i32(graph.is_directed()))
    A = DeviceCSR.from_counts(
        (ne, ne), dt, graph.device,
        lambda st, ip, nnz: nat.call("gsp_line_graph_count", *head, *tail, ip, nnz, st),
        lambda st, ip, ix, d: nat.call("gsp_line_graph_fill_" + nat.suffix(dt), *head, D.indices,
                                       *tail, ip, ix, d, st),
        "line graph")
    return A, sources, targets


class LineGraph(Graph):
    r"""Line graph of a graph (pygsp/graphs/linegraph.py).

    One vertex per edge of ``graph`` (its edge list order); two are linked, with weight 1, when
    their edges share an end.  W = (D != 0)^T (D != 0) - I is built on the device from the edge
    list and the rows of ``graph.D`` (left set, as in the reference).  A self-loop edge has an
    empty column of D, so its vertex carries the single entry -1.  Coordinates are the edges'
    midpoints (0 for a loop), if ``graph`` has coordinates.  The line graph takes ``graph``'s
    dtype and device unless ``dtype`` / ``device`` are given.
    """

    def __init__(self, graph, **kwargs):
        if graph.is_weighted():
            logger.warning("Your graph is weighted, and is considered "
                           "unweighted to build a binary line graph.")
        kwargs.setdefault("dtype", graph.dtype)
        kwargs.setdefault("device", graph.device)
        W, sources, targets = line_graph_adjacency(graph, kwargs["dtype"])
        coords = getattr(graph, "coords", None)
        if coords is not None:
            c = np.asarray(coords)
            s, t = sources.cpu().numpy(), targets.cpu().numpy()
            loop = (s == t).reshape((-1,) + (1,) * (c.ndim - 1))
            # the reference's sparse product: 0 + c[s] + c[t] per edge, nothing for a loop
            coords = np.where(loop, 0, (np.zeros_like(c[s]) + c[s]) + c[t]) / 2
        super().__init__(W, coords=coords, plotting=graph.plotting, **kwargs)
