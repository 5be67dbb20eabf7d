"""Sampled point-cloud graph models (pygsp/graphs/community.py, swissroll.py and
nngraphs/{sphere,cube,twomoons}.py).

Coordinates are drawn on the host with the reference's own generator calls, in its order, so
they equal the reference's bit for bit.  Edges are built on the device:

* ``Community``: intra-community edges by the segmented radius or k-NN search of
  csrc/neighbors.cu (each community one segment of the sorted vertices), or, with
  ``comm_density``, by an exact-size uniform subset of each community's pairs; inter-community
  edges by an exact-size uniform subset of the pairs across communities (``gsp_subset_select``
  in csrc/random_graphs.cu).  The Philox key is ``rng.integers(2**63)`` drawn after the
  coordinates, so the reference's graph and this one share every draw up to the edges.
* ``SwissRoll``: the thresholded Gaussian kernel is a radius graph of the rescaled points.
* ``Sphere``, ``Cube``, ``TwoMoons``: the reference's point clouds through :class:`NNGraph`.

DESIGN.md sections 2 and 4.19 list where the results differ from the reference's.
"""
import math

import numpy as np

from .. import _native as nat
from .. import utils
from .csr import DeviceCSR, row_ids
from .generators import NNGraph, _device_of, _device_points, _gauss_weights_device
from .graph import Graph, _torch_dtype
from .random_graphs import _CHUNK_TARGET, PLAN_COLS, RECT, TRI_STRICT, _assemble

# Grid cap of the subset launches (0: the default shape).  Results do not depend on it.
_MAX_BLOCKS = 0
# The walk of a space draws at a probability that leaves fewer than its target with probability
# below exp(-_MISS_LOG) (a Chernoff bound); a short walk is redrawn with the next key.
_MISS_LOG = math.log(1e12)
_KEY_STEP = 0x9E3779B97F4A7C15
_MAX_ATTEMPTS = 16


# ---------------------------------------------------------------- exact-size subsets ---------
def inflated_probability(n, M):
    """Walk probability of a space of M pairs with target n: the mean n + d of the number of
    candidates K ~ Binomial(M, p) leaves P(K < n) <= exp(-d^2 / (2 (n + d))) = 1e-12; 1 when
    that mean reaches M."""
    if n <= 0:
        return 0.0
    d = _MISS_LOG + math.sqrt(_MISS_LOG * _MISS_LOG + 2.0 * _MISS_LOG * n)
    return 1.0 if n + d >= M else (n + d) / M


def attempt_key(key, attempt):
    """Philox key of the walk of attempt ``attempt`` (the priorities always use ``key``)."""
    return (int(key) + attempt * _KEY_STEP) % 2 ** 64


def subset_plan(spaces, target=None):
    """Chunk plan of the subset walk: (plan (nblk, PLAN_COLS) int64, prob (nblk, 2) float64,
    number of chunks, space_chunk (n_spaces + 1) int64, targets (n_spaces) int64).

    ``spaces`` is a list of (blocks, n): blocks a list of (kind, n_pairs, width, row0, col0) --
    a rectangle (RECT) or a strict lower triangle (TRI_STRICT) of vertex pairs, decoded as the
    SBM plan -- and n <= sum of n_pairs the size of the subset.  A space with n = 0 is not
    walked."""
    target = _CHUNK_TARGET if target is None else target
    plan, prob, space_chunk, targets, cfirst = [], [], [0], [], 0
    for blocks, n in spaces:
        M = sum(int(b[1]) for b in blocks)
        n = int(n)
        if not 0 <= n <= M:
            raise ValueError("a subset of {} pairs out of {} is not possible".format(n, M))
        p = inflated_probability(n, M)
        for kind, n_pairs, width, row0, col0 in blocks:
            if n == 0 or n_pairs == 0:
                continue
            clen = min(max(math.ceil(target / p), 1), int(n_pairs))
            plan.append([n_pairs, clen, cfirst, row0, col0, width, kind, 0])
            prob.append([p, math.log1p(-p) if p < 1 else -math.inf])
            cfirst += -(-int(n_pairs) // clen)
        space_chunk.append(cfirst)
        targets.append(n)
    return (np.array(plan, dtype=np.int64).reshape(-1, PLAN_COLS),
            np.array(prob, dtype=np.float64).reshape(-1, 2), cfirst,
            np.array(space_chunk, dtype=np.int64), np.array(targets, dtype=np.int64))


def subset_device(N, spaces, key, device=None):
    """(rows, cols, attempts): a uniform n-subset of the vertex pairs of every space of
    :func:`subset_plan`, drawn on the device with Philox key ``key`` -- both orientations of
    each pair, 2 sum(n) int32 COO entries, space after space.  A function of (key, spaces)
    only.  ``ValueError`` when the entries would reach 2^31, before anything is drawn."""
    torch = nat.require_cuda()
    dev = _device_of(device)
    plan, prob, n_chunks, space_chunk, targets = subset_plan(spaces)
    total = 2 * int(targets.sum())
    if total >= 2 ** 31:
        raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                         "supported.".format(total))
    with torch.cuda.device(dev):
        rows = torch.empty(total, dtype=torch.int32, device=dev)
        cols = torch.empty(total, dtype=torch.int32, device=dev)
        if total == 0:
            return rows, cols, 0
        st = nat.stream_ptr(dev)
        perm = torch.arange(N, dtype=torch.int32, device=dev)
        plan_t, prob_t = torch.from_numpy(plan).to(dev), torch.from_numpy(prob).to(dev)
        offsets = torch.empty(n_chunks + 1, dtype=torch.int64, device=dev)
        bounds = torch.from_numpy(space_chunk).to(dev)
        for attempt in range(_MAX_ATTEMPTS):
            args = (nat.i64(n_chunks), nat.i64(len(plan)), plan_t, prob_t,
                    nat.u64(attempt_key(key, attempt)))
            nat.call("gsp_sbm_count", *args, offsets, nat.i32(_MAX_BLOCKS), st)
            begin = offsets[bounds].cpu().numpy()
            if (np.diff(begin) >= targets).all():
                break
        else:
            raise nat.NativeError("the subset walk came up short %d times" % _MAX_ATTEMPTS)
        n_cand = int(begin[-1])
        if n_cand >= 2 ** 31:
            raise ValueError("the subset walk drew {} candidates; at most 2^31 - 1 are "
                             "supported".format(n_cand))
        cand_r = torch.empty(n_cand, dtype=torch.int32, device=dev)
        cand_c = torch.empty(n_cand, dtype=torch.int32, device=dev)
        nat.call("gsp_sbm_fill", *args, perm, offsets, cand_r, cand_c, nat.i32(_MAX_BLOCKS), st)
        nat.call("gsp_subset_select", nat.i64(N), nat.i64(n_chunks), offsets,
                 nat.i64(len(targets)), space_chunk, targets, nat.u64(key), cand_r, cand_c, rows,
                 cols, nat.i32(_MAX_BLOCKS), st)
    return rows, cols, attempt


# ---------------------------------------------------------------- segmented searches ---------
def _segment_tables(sizes, dev):
    """(n_seg, seg_start int64, seg_id int32) device tables of consecutive segments."""
    torch = nat.require_cuda()
    sizes = np.asarray(sizes, dtype=np.int64)
    start = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    seg_id = np.repeat(np.arange(sizes.size, dtype=np.int32), sizes)
    return (nat.i64(sizes.size), torch.from_numpy(start).to(dev),
            torch.from_numpy(seg_id).to(dev))


def radius_segments_device(points, sizes, epsilon, p=2, device=None, check=None):
    """Radius neighbourhoods inside segments: the (N, N) DeviceCSR of float64 distances whose
    row i holds the j != i of i's segment with dist(x_i, x_j) <= epsilon (``gsp_radius_*_seg``).
    The segments are consecutive runs of ``sizes`` vertices.  ``check(nnz)`` may refuse the
    size after the count, before the fill."""
    torch = nat.require_cuda()
    dev = _device_of(device)
    pts = _device_points(points, dev)
    n, dim = pts.shape
    cloud = (nat.i64(n), nat.i32(dim), pts, nat.f64(epsilon), nat.f64(p),
             *_segment_tables(sizes, dev))
    return DeviceCSR.from_counts(
        (n, n), torch.float64, dev,
        lambda st, ip, nnz: nat.call("gsp_radius_count_seg", *cloud, ip, nnz, st),
        lambda st, ip, ix, d: nat.call("gsp_radius_fill_seg_f64", *cloud, ip, ix, d, st),
        "graph", check=check)


def knn_segments_device(points, sizes, k, p=2, device=None):
    """(nn, dist), (N, k): the k nearest neighbours of every point inside its segment
    (``gsp_knn_brute_seg``), ascending (distance, id), padded with -1 / 0 where the segment has
    fewer than k other points."""
    torch = nat.require_cuda()
    dev = _device_of(device)
    pts = _device_points(points, dev)
    n, dim = pts.shape
    nn = torch.empty((n, k), dtype=torch.int32, device=dev)
    dist = torch.empty((n, k), dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        nat.call("gsp_knn_brute_seg", nat.i64(n), nat.i32(dim), pts, nat.i32(k), nat.f64(p),
                 *_segment_tables(sizes, dev), nn, dist, nat.stream_ptr(dev))
    return nn, dist


def _entries_check(extra):
    def check(nnz):
        if nnz + extra >= 2 ** 31:
            raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                             "supported.".format(nnz + extra))
    return check


# ---------------------------------------------------------------- models ---------------------
def community_coordinates(node_com, sizes, world_rad, rng):
    """(com_coords, coords) of community.py: the centres on the circle of radius world_rad,
    then one ``rng.uniform(size=(N, 2))`` draw mapped to polar offsets of radius sqrt(size)
    around each vertex's centre -- the reference's per-vertex loop, vectorised, same bits."""
    Nc, N = len(sizes), len(node_com)
    angles = 2 * np.pi * np.arange(1, Nc + 1) / Nc
    com_coords = world_rad * np.stack([np.cos(angles), np.sin(angles)], axis=1).reshape(Nc, 2)
    radius, turn = rng.uniform(size=(N, 2)).T
    offset = np.stack([radius * np.cos(2 * np.pi * turn), radius * np.sin(2 * np.pi * turn)],
                      axis=1)
    return com_coords, com_coords[node_com] + np.sqrt(sizes[node_com])[:, None] * offset


def swissroll_points(N, a, b, dim, noise, srtype, seed):
    """The (dim, N) points x of swissroll.py, with its default_rng(seed) draws in its order."""
    rng = np.random.default_rng(seed)
    y1 = rng.uniform(size=N)
    y2 = rng.uniform(size=N)
    if srtype == "uniform":
        tt = np.sqrt((b * b - a * a) * y1 + a * a)
    else:
        tt = (b - a) * y1 + a
    tt *= np.pi
    if dim == 2:
        x = np.array((tt * np.cos(tt), tt * np.sin(tt)))
    else:
        x = np.array((tt * np.cos(tt), 21 * y2, tt * np.sin(tt)))
    if noise:
        x += rng.normal(size=x.shape)
    return x


def sphere_points(nb_pts, nb_dim, seed):
    """Normal draws of RandomState(seed) normalised row by row, as sphere.py: with the 1-D
    norm of each row, which norm(axis=1) does not reproduce bit for bit."""
    pts = np.random.RandomState(seed).normal(0, 1, (nb_pts, nb_dim))
    for i in range(nb_pts):
        pts[i] /= np.linalg.norm(pts[i])
    return pts


def cube_points(nb_pts, nb_dim, seed):
    """cube.py's points: the unit square (2-D) or nb_pts // 6 points on each face of the unit
    cube in the reference's draw order (3-D)."""
    rs = np.random.RandomState(seed)
    if nb_dim == 2:
        return rs.rand(nb_pts, nb_dim)
    n = nb_pts // 6
    pts = np.zeros((n * 6, 3))
    pts[:n, 1:] = rs.rand(n, 2)
    pts[n:2 * n, :] = np.concatenate((np.ones((n, 1)), rs.rand(n, 2)), axis=1)
    pts[2 * n:3 * n, :] = np.concatenate((rs.rand(n, 1), np.zeros((n, 1)), rs.rand(n, 1)),
                                         axis=1)
    pts[3 * n:4 * n, :] = np.concatenate((rs.rand(n, 1), np.ones((n, 1)), rs.rand(n, 1)),
                                         axis=1)
    pts[4 * n:5 * n, :2] = rs.rand(n, 2)
    pts[5 * n:6 * n, :] = np.concatenate((rs.rand(n, 2), np.ones((n, 1))), axis=1)
    return pts


class Community(Graph):
    r"""Community graph (pygsp/graphs/community.py): Nc communities on a circle of radius
    ``size_ratio * sqrt(N)``, each vertex at a random offset of radius sqrt(community size) from
    its community's centre.

    Intra-community edges: the pairs of a community within ``epsilon`` (default), a uniform
    ``int(comm_density * M_c)``-subset of its M_c pairs, or the union of every vertex's
    ``k_neigh`` nearest neighbours in its community (``k_neigh <= 32``).  Inter-community
    edges: a uniform ``int(world_density * M)``-subset of the M pairs across communities.  Unit
    weights.  Arguments, defaults, ``info``, ``Nc`` and errors are the reference's; the edge
    draws are Philox streams, so sampled edges equal the reference's in law only (DESIGN.md
    section 2).
    """

    def __init__(self, N=256, Nc=None, min_comm=None, min_deg=None, comm_sizes=None,
                 size_ratio=1, world_density=None, comm_density=None, k_neigh=None,
                 epsilon=None, seed=None, **kwargs):
        if Nc is None:
            Nc = int(round(np.sqrt(N) / 2))
        if min_comm is None:
            min_comm = int(round(N / (3 * Nc)))
        if min_deg is not None:
            raise NotImplementedError
        if world_density is None:
            world_density = 1 / N
        if not 0 <= world_density <= 1:
            raise ValueError("World density should be in [0, 1].")
        if epsilon is None:
            epsilon = np.sqrt(2 * np.sqrt(N)) / 2

        self.Nc, self.min_comm, self.comm_sizes = Nc, min_comm, comm_sizes
        self.size_ratio, self.world_density = size_ratio, world_density
        self.comm_density, self.k_neigh, self.epsilon, self.seed = comm_density, k_neigh, \
            epsilon, seed
        rng = np.random.default_rng(seed)
        if min_comm * Nc > N:
            raise ValueError("The constraint on minimum size for communities is unsolvable.")
        info = {"node_com": None, "comm_sizes": None, "world_rad": None,
                "world_density": world_density, "min_comm": min_comm}
        if comm_sizes is None:
            mandatory = np.tile(np.arange(Nc), (min_comm,))
            info["node_com"] = np.sort(np.concatenate((mandatory,
                                                       rng.choice(Nc, N - min_comm * Nc))))
        else:
            if len(comm_sizes) != Nc:
                raise ValueError("There should be Nc community sizes.")
            if np.sum(comm_sizes) != N:
                raise ValueError("The sum of community sizes should be N.")
            info["node_com"] = np.concatenate([[val] * cnt for val, cnt in enumerate(comm_sizes)])
        node_com = np.asarray(info["node_com"], dtype=np.int64)
        info["comm_sizes"] = np.bincount(node_com, minlength=Nc)
        info["world_rad"] = size_ratio * np.sqrt(N)
        if comm_density is not None:
            if not 0 <= comm_density <= 1:
                raise ValueError("comm_density should be between 0 and 1.")
            info["comm_density"] = comm_density
        elif k_neigh is not None:
            if k_neigh < 0:
                raise ValueError("k_neigh cannot be negative.")
            if k_neigh > 32:
                raise ValueError("k_neigh must be at most 32 (the device k-NN search).")
            info["k_neigh"] = k_neigh
        else:
            info["epsilon"] = epsilon

        info["com_coords"], coords = community_coordinates(node_com, info["comm_sizes"],
                                                           info["world_rad"], rng)
        sizes = info["comm_sizes"]
        key = int(rng.integers(2 ** 63))

        torch = nat.require_cuda()
        dev = _device_of(kwargs.get("device"))
        dt = _torch_dtype(torch, kwargs.get("dtype"))
        start = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        M = (N ** 2 - np.sum(sizes ** 2)) / 2
        n_inter = int(world_density * M)
        inter = [(RECT, int(sizes[a] * sizes[b]), int(sizes[b]), int(start[a]), int(start[b]))
                 for a in range(Nc) for b in range(a)]
        spaces = [(inter, n_inter)]
        rows, cols = [], []
        if comm_density is not None:
            spaces = [([(TRI_STRICT, int(s * (s - 1) // 2), int(s), int(start[c]),
                         int(start[c]))], int(comm_density * (s * (s - 1) / 2)))
                      for c, s in enumerate(sizes)] + spaces
        elif k_neigh is not None:
            k = min(int(k_neigh), int(sizes.max()) - 1) if N else 0
            if k >= 1:
                nn, _ = knn_segments_device(coords, sizes, k, 2, dev)
                keep = nn.reshape(-1) >= 0
                src = torch.arange(N, device=dev).repeat_interleave(k)[keep]
                directed = DeviceCSR.from_coo(src, nn.reshape(-1)[keep],
                                              torch.ones(int(keep.sum().item()), dtype=dt,
                                                         device=dev), (N, N))
                S = directed.symmetrize("maximum")
                rows.append(row_ids(S.indptr).int())
                cols.append(S.indices)
        else:
            D = radius_segments_device(coords, sizes, epsilon, 2, dev,
                                       check=_entries_check(2 * n_inter))
            rows.append(row_ids(D.indptr).int())
            cols.append(D.indices)
        sr, sc, self._attempts = subset_device(N, spaces, key, dev)
        rows.append(sr)
        cols.append(sc)
        rows, cols = torch.cat(rows), torch.cat(cols)
        if rows.numel() >= 2 ** 31:
            raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                             "supported.".format(rows.numel()))
        W = _assemble(rows, cols, N, dt)
        self.info = info
        super().__init__(W, coords=coords, **kwargs)

    def _get_extra_repr(self):
        attrs = {"Nc": self.Nc, "min_comm": self.min_comm, "comm_sizes": self.comm_sizes,
                 "size_ratio": f"{self.size_ratio:.2f}",
                 "world_density": f"{self.world_density:.2f}"}
        if self.comm_density is not None:
            attrs["comm_density"] = f"{self.comm_density:.2f}"
        elif self.k_neigh is not None:
            attrs["k_neigh"] = self.k_neigh
        else:
            attrs["epsilon"] = f"{self.epsilon:.2f}"
        attrs["seed"] = self.seed
        return attrs


# exp(-x) is 0 in double beyond this x: the radius of SwissRoll(thresh <= 0)
_EXP_UNDERFLOW = 746.0
# relative enlargement of the squared radius: covers the rounding of the distance and of the
# exponential, the weight predicate then decides exactly
_RADIUS_MARGIN = 1e-9


class SwissRoll(Graph):
    r"""Sampled Swiss roll manifold (pygsp/graphs/swissroll.py).

    W_ij = exp(-d_ij^2 / (2 s^2)) for i != j, entries below ``thresh`` dropped, over the
    rescaled points ``coords = utils.rescale_center(x).T``.  Built as a radius graph of radius
    sqrt(-2 s^2 ln(thresh)) (capped at the exponential's underflow for ``thresh <= 0``) with
    distances from direct differences, then the weight predicate.  ``dim`` must be 2 or 3 and
    ``srtype`` 'uniform' or 'classic' (``ValueError``).
    """

    def __init__(self, N=400, a=1, b=4, dim=3, thresh=1e-6, s=None, noise=False,
                 srtype="uniform", seed=None, **kwargs):
        if s is None:
            s = np.sqrt(2.0 / N)
        if dim not in (2, 3):
            raise ValueError("dim must be 2 or 3, not {}.".format(dim))
        if srtype not in ("uniform", "classic"):
            raise ValueError("Unknown srtype {}.".format(srtype))
        self.a, self.b, self.dim, self.thresh, self.s = a, b, dim, thresh, s
        self.noise, self.srtype, self.seed = noise, srtype, seed

        self.x = x = swissroll_points(N, a, b, dim, noise, srtype, seed)
        coords = utils.rescale_center(x)

        torch = nat.require_cuda()
        dev = _device_of(kwargs.get("device"))
        dt = _torch_dtype(torch, kwargs.get("dtype"))
        sigma = 2.0 * s ** 2
        scaled = -math.log(thresh) if thresh > 0 else _EXP_UNDERFLOW
        eps2 = max(sigma * min(scaled, _EXP_UNDERFLOW), 0.0) * (1.0 + _RADIUS_MARGIN)
        D = radius_segments_device(coords.T, [N], math.sqrt(eps2), 2, dev)
        W64 = _gauss_weights_device(D, sigma, torch.float64)
        W64.data.masked_fill_(W64.data < thresh, 0.0)
        W = DeviceCSR(W64.indptr, W64.indices, W64.data.to(dt), W64.shape).eliminate_zeros()
        plotting = {"vertex_size": 60, "limits": np.array([-1, 1, -1, 1, -1, 1]),
                    "elevation": 15, "azimuth": -90, "distance": 7}
        super().__init__(W, coords=coords.T, plotting=plotting, **kwargs)

    def _get_extra_repr(self):
        return {"a": self.a, "b": self.b, "dim": self.dim, "thresh": f"{self.thresh:.0e}",
                "s": f"{self.s:.2f}", "noise": self.noise, "srtype": self.srtype,
                "seed": self.seed}


def _nn_repr(G):
    return {"NNtype": G.NNtype, "use_flann": G.use_flann, "center": G.center,
            "rescale": G.rescale, "k": G.k, "sigma": f"{G.sigma:.2f}",
            "epsilon": f"{G.epsilon:.2f}", "symmetrize_type": G.symmetrize_type,
            "dist_type": G.dist_type, "order": None}


class Sphere(NNGraph):
    r"""Points drawn uniformly on the unit sphere (pygsp/graphs/nngraphs/sphere.py): normal
    draws of ``RandomState(seed)`` normalised row by row, then the 10-NN graph."""

    def __init__(self, radius=1, nb_pts=300, nb_dim=3, sampling="random", seed=None, **kwargs):
        self.radius, self.nb_pts, self.nb_dim = radius, nb_pts, nb_dim
        self.sampling, self.seed = sampling, seed
        if sampling != "random":
            raise ValueError(f"Unknown sampling {sampling}")
        super().__init__(Xin=sphere_points(nb_pts, nb_dim, seed), k=10, center=False, rescale=False,
                         plotting={"vertex_size": 80}, **kwargs)

    def _get_extra_repr(self):
        attrs = {"radius": f"{self.radius:.2f}", "nb_pts": self.nb_pts, "nb_dim": self.nb_dim,
                 "sampling": self.sampling, "seed": self.seed}
        attrs.update(_nn_repr(self))
        return attrs


class Cube(NNGraph):
    r"""Points drawn on the unit square (2-D) or on the six faces of the unit cube, nb_pts // 6
    per face in the reference's order (3-D) (pygsp/graphs/nngraphs/cube.py), then the 10-NN
    graph.  ``nb_dim > 3``: ``NotImplementedError``; ``nb_dim`` 1 or an unknown ``sampling``:
    ``ValueError``."""

    def __init__(self, radius=1, nb_pts=300, nb_dim=3, sampling="random", seed=None, **kwargs):
        self.radius, self.nb_pts, self.nb_dim = radius, nb_pts, nb_dim
        self.sampling, self.seed = sampling, seed
        if nb_dim > 3:
            raise NotImplementedError("Dimension > 3 not supported yet!")
        if sampling != "random":
            raise ValueError("Unknown sampling !")
        if nb_dim not in (2, 3):
            raise ValueError("nb_dim must be 2 or 3, not {}.".format(nb_dim))
        super().__init__(Xin=cube_points(nb_pts, nb_dim, seed), k=10, center=False, rescale=False,
                         plotting={"vertex_size": 80, "elevation": 15, "azimuth": 0,
                                   "distance": 9}, **kwargs)

    def _get_extra_repr(self):
        attrs = {"radius": f"{self.radius:.2f}", "nb_pts": self.nb_pts, "nb_dim": self.nb_dim,
                 "sampling": self.sampling, "seed": self.seed}
        attrs.update(_nn_repr(self))
        return attrs


class TwoMoons(NNGraph):
    r"""Two moons (pygsp/graphs/nngraphs/twomoons.py), the 5-NN graph with ``sigma=sigmag``.

    'synthesized': N // 2 and N - N // 2 points on two noisy half circles; both moons are drawn
    from ``default_rng(seed)``, so with a seed they share their draws, as in the reference.
    'standard' reads the reference's two_moons point cloud, a data file this package does not
    ship: ``NotImplementedError``.
    """

    def __init__(self, moontype="standard", dim=2, sigmag=0.05, N=400, sigmad=0.07,
                 distance=0.5, seed=None, **kwargs):
        self.moontype, self.dim, self.sigmag, self.sigmad = moontype, dim, sigmag, sigmad
        self.distance, self.seed = distance, seed
        if moontype == "standard":
            raise NotImplementedError("TwoMoons('standard') needs the reference's two_moons "
                                      "data file, which is not shipped; use 'synthesized'.")
        if moontype != "synthesized":
            raise ValueError(f"Unknown moontype {moontype}")
        N1 = N // 2
        N2 = N - N1
        Xin = np.concatenate((self._create_arc_moon(N1, sigmad, distance, 1, seed),
                              self._create_arc_moon(N2, sigmad, distance, 2, seed)))
        self.labels = np.concatenate((np.zeros(N1), np.ones(N2)))
        super().__init__(Xin=Xin, sigma=sigmag, k=5, center=False, rescale=False,
                         plotting={"vertex_size": 30}, **kwargs)

    @staticmethod
    def _create_arc_moon(N, sigmad, distance, number, seed):
        rng = np.random.default_rng(seed)
        phi = rng.uniform(size=(N, 1)) * np.pi
        rb = sigmad * rng.normal(size=(N, 1))
        ab = rng.uniform(size=(N, 1)) * 2 * np.pi
        b = rb * np.exp(1j * ab)
        bx, by = np.real(b), np.imag(b)
        if number == 1:
            return np.concatenate((np.cos(phi) + bx + 0.5,
                                   -np.sin(phi) + by - (distance - 1) / 2.0), axis=1)
        return np.concatenate((np.cos(phi) + bx - 0.5, np.sin(phi) + by + (distance - 1) / 2.0),
                              axis=1)

    def _get_extra_repr(self):
        attrs = {"moontype": self.moontype, "dim": self.dim, "sigmag": f"{self.sigmag:.2f}",
                 "sigmad": f"{self.sigmad:.2f}", "distance": f"{self.distance:.2f}",
                 "seed": self.seed}
        attrs.update(_nn_repr(self))
        return attrs
