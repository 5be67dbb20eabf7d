"""Vertex coordinates: set_coordinates and the Fruchterman-Reingold spring layout.

Mirror of ``pygsp.graphs._layout`` (``set_coordinates``, _layout.py:5-119, and
``_fruchterman_reingold``, :121-233), mixed into :class:`Graph`.  Same kinds, keyword arguments,
exceptions and log message.  ``coords`` is a host NumPy array, as everywhere in the package.

The host kinds ('line1D', 'line2D', 'ring2D', 'random2D', 'random3D', 'community2D') are the
reference's NumPy expressions with the same seeded generator, so they are bit-identical to it.
The eigenmaps are columns of this engine's own Fourier basis (graphs/fourier.py).  The spring
layout draws the reference's seeded start on the host, runs every iteration on the device
(``gsp_spring_layout_*``, csrc/layout.cu: an all-pairs float64 kernel) at the reference's exact
temperatures, and rescales the result on the host with the reference's operations.

``set_coordinates('spring', repulsion='barnes_hut', theta=0.5)`` replaces only the repulsion sum,
which costs O(N^2) per iteration, by a Barnes-Hut walk of a Morton-ordered radix tree rebuilt on
the device every iteration (``gsp_spring_layout_bh_*``, csrc/barnes_hut.cu, DESIGN.md section
4.24): O(N log N), for dim 1, 2 or 3.  A cell is taken as one monopole when the diagonal of its
points' bounding box is at most ``theta`` times the distance from the vertex to that box (and the
distance is at least 0.01), so each vertex's repulsion is within a proven bound of the exact sum
(DESIGN.md section 4.24); ``theta=0`` opens every cell of distinct points.  The attraction,
the move, the cooling schedule, ``fixed``, ``pos``, ``k``, the seeded start and the rescale are
unchanged, and ``repulsion='exact'``, the default, is the all-pairs kernel.

Differences from the reference (DESIGN.md section 2): the spring layout's float64 sums run in
another order (the iteration is chaotic, so a 50-iteration layout differs from the reference's
by more than rounding, while each single step agrees to rounding); the sign of each eigenmap
column is the engine's; a graph without ``info`` raises ``AttributeError`` from
'community2D' explicitly, and missing ``comm_sizes`` are counted with ``np.bincount`` (the
reference would fail on an unimported ``Counter``); no binary adjacency matrix ``A`` is built.
"""
import numpy as np

from .. import _native as nat


class LayoutMixIn:

    def set_coordinates(self, kind="spring", seed=None, **kwargs):
        r"""Set the vertices' coordinates (their position when plotting).

        Parameters
        ----------
        kind : string or array_like
            An array of size N, Nx2 or Nx3 sets the coordinates directly.  Otherwise the name of
            a layout: 'community2D', 'random2D', 'random3D', 'ring2D', 'line1D', 'line2D',
            'spring' (default), 'laplacian_eigenmap2D', 'laplacian_eigenmap3D'.
        seed : int
            Seed of the random generator for 'random2D', 'random3D', 'community2D' and 'spring'.
        kwargs : dict
            Arguments of the Fruchterman-Reingold layout when kind is 'spring': ``dim`` (2),
            ``k`` (None: sqrt(1/N)), ``pos`` (None), ``fixed`` ([]), ``iterations`` (50),
            ``scale`` (1.0) and ``center`` (None: the origin).  Two more select the repulsion
            sum: ``repulsion`` ('exact', the default: all pairs, O(N^2) per iteration; or
            'barnes_hut': a Barnes-Hut tree walk, O(N log N), approximate within a proven
            bound, dim 1, 2 or 3 only) and ``theta`` (0.5; 'barnes_hut' only: a cell is one
            monopole when its bounding box's diagonal is at most ``theta`` times its distance
            from the vertex, so a smaller ``theta`` is slower and closer to the exact sum).
            An unknown ``repulsion``, ``theta`` with 'exact', a negative or non-finite
            ``theta``, and a ``dim`` other than 1, 2, 3 or a non-finite ``pos`` with
            'barnes_hut' raise ``ValueError``.
        """
        if not isinstance(kind, str):
            coords = np.asanyarray(kind).squeeze()
            check_1d = coords.ndim == 1
            check_2d_3d = coords.ndim == 2 and 2 <= coords.shape[1] <= 3
            if coords.shape[0] != self.N or not (check_1d or check_2d_3d):
                raise ValueError("Expecting coordinates to be of size N, Nx2, or Nx3.")
            self.coords = coords
        elif kind == "line1D":
            self.coords = np.arange(self.N)
        elif kind == "line2D":
            self.coords = np.stack([np.arange(self.N), np.zeros(self.N)], axis=1)
        elif kind == "ring2D":
            angle = np.arange(self.N) * 2 * np.pi / self.N
            self.coords = np.stack([np.cos(angle), np.sin(angle)], axis=1)
        elif kind == "random2D":
            self.coords = np.random.default_rng(seed).uniform(size=(self.N, 2))
        elif kind == "random3D":
            self.coords = np.random.default_rng(seed).uniform(size=(self.N, 3))
        elif kind == "spring":
            self.coords = self._fruchterman_reingold(seed=seed, **kwargs)
        elif kind == "community2D":
            self.coords = self._community_coordinates(seed)
        elif kind == "laplacian_eigenmap2D":
            self.compute_fourier_basis(n_eigenvectors=3)
            self.coords = self.U[:, 1:3]
        elif kind == "laplacian_eigenmap3D":
            self.compute_fourier_basis(n_eigenvectors=4)
            self.coords = self.U[:, 1:4]
        else:
            raise ValueError(f"Unexpected argument kind={kind}.")

    def _community_coordinates(self, seed):
        """Communities on a circle of radius info['world_rad'], each vertex at a random offset of
        radius sqrt(community size) from its community's centre (_layout.py:64-111)."""
        if not hasattr(self, "info"):
            raise AttributeError("Missing arguments to the graph to be able to compute "
                                 "community coordinates: the graph has no info.")
        info = self.info
        node_com = np.asarray(info["node_com"])
        if "world_rad" not in info:
            info["world_rad"] = np.sqrt(self.N)
        if "comm_sizes" not in info:
            info["comm_sizes"] = np.bincount(node_com)
        n_com = info["comm_sizes"].shape[0]
        angles = 2 * np.pi * np.arange(1, n_com + 1) / n_com
        info["com_coords"] = info["world_rad"] * np.stack([np.cos(angles), np.sin(angles)],
                                                          axis=1)
        rng = np.random.default_rng(seed)
        radius, turn = rng.uniform(size=(self.N, 2)).T
        offset = np.stack([radius * np.cos(2 * np.pi * turn), radius * np.sin(2 * np.pi * turn)],
                          axis=1)
        comm_rad = np.sqrt(info["comm_sizes"][node_com])
        return info["com_coords"][node_com] + comm_rad[:, None] * offset

    def _fruchterman_reingold(self, dim=2, k=None, pos=None, fixed=[], iterations=50,
                              scale=1.0, center=None, seed=None, repulsion="exact", theta=None):
        """The reference's argument handling (_layout.py:136-166) around the device layout."""
        _repulsion_theta(repulsion, theta, dim)
        if center is None:
            center = np.zeros((1, dim))
        if np.shape(center)[1] != dim:
            self.logger.error("Spring coordinates: center has wrong size.")
            center = np.zeros((1, dim))

        if pos is None:
            dom_size = 1
            start = np.random.default_rng(seed).uniform(size=(self.N, dim))
        else:
            # the reference's start is row i of pos for every vertex i (:148-153)
            dom_size = np.max(pos)
            given = np.asanyarray(pos, dtype=np.float64)
            start = np.empty((self.N, dim))
            start[:] = given[:self.N, None] if given.ndim == 1 else given[:self.N]

        if k is None and len(fixed) > 0:
            k = dom_size / np.sqrt(self.N)
        if k is None:
            k = np.sqrt(1.0 / self.N)

        pos = _spring_layout(self, start, k, iterations, fixed, repulsion=repulsion, theta=theta)
        if len(fixed) == 0:
            pos = _rescale_layout(pos, scale=scale) + center
        return pos


def _temperatures(iterations):
    """The reference's cooling schedule (_layout.py:190-191, 217) in Python floats."""
    t = 0.1
    dt = t / float(iterations + 1)
    out = []
    for _ in range(iterations):
        out.append(t)
        t -= dt
    return np.array(out, dtype=np.float64)


def _repulsion_theta(repulsion, theta, dim):
    """The ``theta`` of a Barnes-Hut repulsion (0.5 by default), None for the exact one; raises
    ``ValueError`` on an unknown ``repulsion``, a ``theta`` given with 'exact', a negative or
    non-finite ``theta`` and a Barnes-Hut ``dim`` other than 1, 2, 3."""
    if repulsion == "exact":
        if theta is not None:
            raise ValueError("theta applies only to repulsion='barnes_hut'.")
        return None
    if repulsion != "barnes_hut":
        raise ValueError("Unexpected argument repulsion=%r: 'exact' or 'barnes_hut'." % (repulsion,))
    theta = 0.5 if theta is None else float(theta)
    if not (np.isfinite(theta) and theta >= 0):
        raise ValueError("theta must be finite and >= 0, got %r." % (theta,))
    if dim not in (1, 2, 3):
        raise ValueError("repulsion='barnes_hut' takes dim 1, 2 or 3, got %r." % (dim,))
    return theta


def _spring_inputs(G, pos, fixed, repulsion="exact", theta=None):
    pos = np.ascontiguousarray(pos, dtype=np.float64)
    theta = _repulsion_theta(repulsion, theta, pos.shape[1] if pos.ndim == 2 else None)
    if theta is not None and not np.isfinite(pos).all():
        raise ValueError("repulsion='barnes_hut' needs finite start positions.")
    torch = nat.require_cuda()
    pos = torch.as_tensor(pos, device=G.device)
    mask = None
    if len(fixed) > 0:
        mask = np.isin(np.arange(G.N), np.asarray(list(fixed))).astype(np.uint8)
        mask = torch.as_tensor(mask, device=G.device)
    return torch, pos.contiguous(), mask, theta


def _spring_layout(G, start, k, iterations, fixed, keep_states=False, *, repulsion="exact",
                   theta=None):
    """``iterations`` spring iterations on the device from ``start`` (N, dim).  Returns the final
    positions (host float64), and with ``keep_states`` also the (iterations, N, dim) positions
    after every iteration.  ``repulsion`` and ``theta`` are those of ``set_coordinates``."""
    torch, pos, mask, theta = _spring_inputs(G, start, fixed, repulsion, theta)
    n, dim = pos.shape
    temps = _temperatures(int(iterations))
    states = None
    if keep_states:
        states = torch.empty((len(temps), n, dim), dtype=torch.float64, device=G.device)
    W = G.W
    args = (nat.i64(n), nat.i32(dim), W.indptr, W.indices, W.data, nat.f64(k),
            nat.i32(len(temps)), temps, mask, pos, states)
    if theta is None:
        G._call("gsp_spring_layout", *args)
    else:
        G._call("gsp_spring_layout_bh", *args, nat.f64(theta))
    out = pos.cpu().numpy()
    return (out, states.cpu().numpy()) if keep_states else out


def _spring_step(G, pos, k, t, fixed=(), *, repulsion="exact", theta=None):
    """One spring iteration at temperature ``t`` from the positions ``pos`` (N, dim) on the
    device; returns the new positions (host float64)."""
    torch, cur, mask, theta = _spring_inputs(G, pos, fixed, repulsion, theta)
    nxt = torch.empty_like(cur)
    W = G.W
    args = (nat.i64(cur.shape[0]), nat.i32(cur.shape[1]), W.indptr, W.indices, W.data,
            nat.f64(k), nat.f64(t), mask, cur, nxt)
    if theta is None:
        G._call("gsp_spring_step", *args)
    else:
        G._call("gsp_spring_step_bh", *args, nat.f64(theta))
    return nxt.cpu().numpy()


def _rescale_layout(pos, scale=1):
    """Centre each axis and scale by the largest coordinate (_layout.py:222-233), in place."""
    lim = 0
    for i in range(pos.shape[1]):
        pos[:, i] -= pos[:, i].mean()
        lim = max(pos[:, i].max(), lim)
    for i in range(pos.shape[1]):
        pos[:, i] *= scale / lim
    return pos
