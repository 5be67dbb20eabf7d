"""``Graph``: the reference's graph object with its sparse algebra in HBM.

Mirror of the part of ``pygsp.graphs.Graph`` that the Chebyshev filtering path
uses (pygsp/graphs/graph.py:98-176 constructor, :510-630 compute_laplacian,
:632-640 _check_signal, :729-838 d / dw, :840-960 lmax / estimate_lmax /
_get_upper_bound, :368-405 is_directed), through ``FourierMixIn``
(graphs/fourier.py) of the Fourier basis, through ``DifferenceMixIn``
(graphs/difference.py) of the differential operator, ``get_edge_list`` and
``dirichlet_energy``, and through ``ConnectivityMixIn`` (graphs/connectivity.py) of
``is_connected``, ``extract_components``, ``subgraph``, ``set_signal`` and
``is_weighted``, and through ``LayoutMixIn`` (graphs/layout.py) of ``set_coordinates``.  Same
constructor signature, same attributes, same
exceptions and log messages; the adjacency, the Laplacian and every vector
derived from them live on the GPU and are produced by the kernels of
``libgspb200`` (csrc/graph.cu, csrc/lanczos.cu, csrc/difference.cu,
csrc/connectivity.cu, csrc/layout.cu).  Out of
scope here, as in SURVEY.md section 2: plotting, IO.
"""
import numpy as np
from scipy import sparse

from .. import _native as nat
from .. import utils
from .connectivity import ConnectivityMixIn
from .csr import DeviceCSR, index32
from .difference import DifferenceMixIn
from .fourier import FourierMixIn
from .layout import LayoutMixIn

_LAP = {"combinatorial": 0, "normalized": 1}


class Graph(FourierMixIn, DifferenceMixIn, ConnectivityMixIn, LayoutMixIn):
    r"""Graph defined by a (weighted) adjacency matrix.

    Parameters
    ----------
    adjacency : sparse matrix, array_like, DeviceCSR or (indptr, indices, data)
        Square adjacency.  Host inputs are converted to CSR (duplicates summed,
        columns sorted) and uploaded; a ``DeviceCSR`` / tensor triple is used
        in place (it must be canonical CSR).
    lap_type : {'combinatorial', 'normalized'}
    coords : array_like, optional
    plotting : dict, optional (kept for signature compatibility)
    dtype : numpy/torch floating dtype, keyword only
        Arithmetic type of the engine: float32 (default) or float64.  The
        reference computes in float64; float64 here reproduces its results to
        round-off, float32 to 1e-5 (normwise).
    device : torch device, keyword only (default: current CUDA device)
    """

    def __init__(self, adjacency, lap_type="combinatorial", coords=None, plotting={},
                 *, dtype=None, device=None):
        torch = nat.require_cuda()
        self.logger = utils.build_logger(__name__)
        self.device = torch.device(device if device is not None
                                   else "cuda:%d" % torch.cuda.current_device())
        self.dtype = _torch_dtype(torch, dtype)
        self._sfx = nat.suffix(self.dtype)

        if isinstance(adjacency, DeviceCSR):
            W = adjacency
        elif isinstance(adjacency, tuple) and len(adjacency) == 3 and torch.is_tensor(adjacency[2]):
            indptr, indices, data = adjacency
            n = indptr.numel() - 1
            W = DeviceCSR(indptr, indices, data, (n, n))
        else:
            if not sparse.issparse(adjacency):
                adjacency = np.asanyarray(adjacency)
            if adjacency.ndim != 2 or adjacency.shape[0] != adjacency.shape[1]:
                raise ValueError("Adjacency: must be a square matrix.")
            host = sparse.csr_matrix(adjacency)          # format conversion only
            if not host.has_canonical_format:
                host = host.copy()
                host.sum_duplicates()
            W = DeviceCSR.from_scipy(host, self.dtype, self.device)
        if W.shape[0] != W.shape[1]:
            raise ValueError("Adjacency: must be a square matrix.")
        if W.data.dtype != self.dtype:
            W = DeviceCSR(W.indptr, W.indices, W.data.to(self.dtype), W.shape)
        W = DeviceCSR(W.indptr.to(self.device, torch.int32).contiguous(),
                      index32(W.indices, W.shape[1], self.device),
                      W.data.to(self.device).contiguous(), W.shape)
        self.n_vertices = W.shape[0]

        stats = self._inspect(W)
        if stats[5] or stats[6]:
            raise ValueError("Adjacency: CSR columns must be sorted, unique and in range.")
        if stats[0]:
            raise ValueError("Adjacency: there is a Not a Number (NaN).")
        if stats[1]:
            raise ValueError("Adjacency: there is an infinite value.")
        if stats[3]:
            self.logger.warning("Adjacency: there are self-loops (non-zeros on the diagonal). "
                                "The Laplacian will not see them.")
        if stats[2]:
            self.logger.warning("Adjacency: there are negative edge weights.")
        if stats[4]:                                     # graph.py:128 eliminate_zeros()
            W = W.eliminate_zeros()
        self._adjacency = W
        self._n_loops = int(stats[3])

        self._directed = None
        self._connected = None
        if self.is_directed():
            self.n_edges = W.nnz
        else:
            self.n_edges = (W.nnz - self._n_loops) // 2 + self._n_loops

        if coords is not None:
            self.coords = np.asanyarray(coords)
        self.plotting = dict(plotting)
        self.signals = dict()

        self._d = None
        self._dw = None
        self._dw_dev = None
        self._d_dev = None
        self._Wt = None
        self._Ws = None
        self._lmax = None
        self._lmax_method = None
        self._lanczos_steps = None
        self._clear_fourier_basis()
        self._D = None

        self.lap_type = lap_type
        self.compute_laplacian(lap_type)
        self.Ne = self.n_edges

    @classmethod
    def from_coo(cls, rows, cols, vals, n_vertices, lap_type="combinatorial", **kwargs):
        """Graph from COO triplets already in HBM (integer rows / cols, float values).

        What ``sparse.csr_matrix(coo)`` does at graph.py:109 -- sort by (row, col), sum
        duplicates in the order given -- runs on the device (:meth:`DeviceCSR.from_coo`); no
        host matrix exists.  An index outside [0, n_vertices) raises ``NativeError``.
        """
        torch = nat.require_cuda()
        dt = _torch_dtype(torch, kwargs.get("dtype", vals.dtype if vals.dtype in
                                            (torch.float32, torch.float64) else None))
        W = DeviceCSR.from_coo(rows, cols, vals.to(dt), (n_vertices, n_vertices))
        kwargs.setdefault("dtype", dt)
        kwargs.setdefault("device", vals.device)
        return cls(W, lap_type=lap_type, **kwargs)

    # ------------------------------------------------------------------ basics
    @property
    def N(self):
        return self.n_vertices

    def __repr__(self):
        return "{}(n_vertices={}, n_edges={})".format(type(self).__name__, self.n_vertices,
                                                      self.n_edges)

    @property
    def W(self):
        r"""Weighted adjacency matrix (a :class:`DeviceCSR`)."""
        return self._adjacency

    @W.setter
    def W(self, value):
        raise AttributeError("In-place modification of the graph is not supported. "
                             "Create another Graph object.")

    def _stream(self):
        return nat.stream_ptr(self.device)

    def _call(self, name, *args):
        torch = nat.require_cuda()
        with torch.cuda.device(self.device):
            nat.call(name + "_" + self._sfx, *args, self._stream())

    def _inspect(self, W):
        torch = nat.require_cuda()
        stats = torch.zeros(8, dtype=torch.int64, device=self.device)
        self._call("gsp_csr_inspect", nat.i64(W.shape[0]), W.indptr, W.indices, W.data, stats)
        return stats.cpu().numpy()

    def has_loops(self):
        return self._n_loops > 0

    def is_directed(self):
        r"""True iff W differs from its transpose (cached; graph.py:368-405)."""
        if self._directed is None:
            torch = nat.require_cuda()
            W = self._adjacency
            count = torch.zeros(1, dtype=torch.int64, device=self.device)
            self._call("gsp_csr_asymmetry", nat.i64(self.n_vertices), W.indptr, W.indices,
                       W.data, count)
            self._directed = bool(count.item() != 0)
        return self._directed

    # ---------------------------------------------------- symmetric part, degree
    def _transpose(self):
        if self._Wt is None:
            self._Wt = self._adjacency.transpose()
        return self._Wt

    def _symmetric_adjacency(self):
        """W for an undirected graph, (W + W^T)/2 otherwise (graph.py:613-616)."""
        if not self.is_directed():
            return self._adjacency
        if self._Ws is None:
            self._Ws = self._adjacency.symmetrize("average", self._transpose())
        return self._Ws

    def _degrees(self):
        if self._dw_dev is None:
            torch = nat.require_cuda()
            W, n = self._adjacency, self.n_vertices
            dw = torch.empty(n, dtype=torch.float64, device=self.device)
            d = torch.empty(n, dtype=torch.float64, device=self.device)
            if self.is_directed():
                Wt = self._transpose()
                self._call("gsp_degree", nat.i64(n), W.indptr, W.data, Wt.indptr, Wt.data, dw, d)
            else:
                self._call("gsp_degree", nat.i64(n), W.indptr, W.data, None, None, dw, d)
            self._dw_dev, self._d_dev = dw, d
        return self._dw_dev, self._d_dev

    @property
    def dw(self):
        r"""Weighted degree (graph.py:783-838): sum_j W[j,i], or (in+out)/2 if directed."""
        if self._dw is None:
            self._dw = self._degrees()[0].cpu().numpy()
        return self._dw

    @property
    def d(self):
        r"""Number of neighbours (graph.py:729-781); (in+out)/2 if directed."""
        if self._d is None:
            d = self._degrees()[1].cpu().numpy()
            self._d = d if self.is_directed() else d.astype(np.int32)
        return self._d

    # ------------------------------------------------------------------ Laplacian
    def compute_laplacian(self, lap_type="combinatorial"):
        r"""Build the graph Laplacian ``self.L`` on the device (graph.py:510-630).

        combinatorial: L = D - W;  normalized: L = I - D^-1/2 W D^-1/2, where a
        directed W is first replaced by (W + W^T)/2.  ``L.indptr`` /
        ``L.indices`` equal SciPy's bit for bit: sorted rows, the diagonal
        merged in place, exact zeros (isolated vertices) not stored.
        """
        if lap_type not in _LAP:
            raise ValueError("Unknown Laplacian type {}".format(lap_type))
        if lap_type != self.lap_type:
            # the reference forgets _lmax_method here, so that G.lmax then returns
            # None (SURVEY.md 3.5); both are reset in this implementation.  The Fourier
            # basis and the differential operator of the old Laplacian go too
            # (graph.py:605-609).
            self._lmax = None
            self._lmax_method = None
            self._clear_fourier_basis()
            self._D = None
        self.lap_type = lap_type

        Ws, n = self._symmetric_adjacency(), self.n_vertices
        dw = self._degrees()[0]
        args = (nat.i64(n), Ws.indptr, Ws.indices, Ws.data, dw, nat.i32(_LAP[lap_type]))
        self.L = DeviceCSR.from_counts(
            (n, n), self.dtype, self.device,
            lambda st, lp, nnz: nat.call("gsp_laplacian_count_" + self._sfx, *args, lp, nnz, st),
            lambda st, lp, li, ld: nat.call("gsp_laplacian_fill_" + self._sfx, *args, lp, li, ld,
                                            st),
            "Laplacian")

    def _check_signal(self, s):
        r"""Validate a signal's first dimension (graph.py:632-640)."""
        torch = nat.require_cuda()
        if not torch.is_tensor(s):
            s = np.asanyarray(s)
        if s.shape[0] != self.n_vertices:
            raise ValueError("First dimension must be the number of vertices "
                             "G.N = {}, got {}.".format(self.N, tuple(s.shape)))
        return s

    # ------------------------------------------------------------------------ lmax
    @property
    def lmax(self):
        r"""Largest eigenvalue of the Laplacian (estimated lazily, with a warning)."""
        if self._lmax is None:
            self.logger.warning("The largest eigenvalue G.lmax is not available, we need to "
                                "estimate it. Explicitly call G.estimate_lmax() or "
                                "G.compute_fourier_basis() once beforehand to suppress the "
                                "warning.")
            self.estimate_lmax()
        return self._lmax

    def estimate_lmax(self, method="lanczos", *, seed=0):
        r"""Estimate the largest eigenvalue of L (cached per method; graph.py:858-931).

        'lanczos' runs a device Lanczos recurrence on the SpMV kernel until the
        Ritz residual is below 5e-3 |theta| (the reference's ARPACK tolerance)
        and returns 1.01 * theta; 'bounds' returns the algebraic upper bound.
        Unlike the reference (unseeded ARPACK start vector) the result is
        reproducible: the start vector is a counter-based function of ``seed``.
        """
        if method == self._lmax_method:
            return
        if method == "lanczos":
            theta = self._lanczos(tol=5e-3, seed=seed)
            bound = self._get_upper_bound()
            slack = 1e-12 if self.dtype == nat.require_cuda().float64 else 1e-5 * abs(bound)
            assert not theta > bound + slack, (theta, bound)
            self._lmax = theta * 1.01
        elif method == "bounds":
            self._lmax = self._get_upper_bound()
        else:
            raise ValueError("Unknown method {}".format(method))
        self._lmax_method = method

    def _lanczos(self, tol, seed, max_steps=400, polish_steps=60):
        """Largest Ritz value of L.

        Stopping rule of the reference (ARPACK, graph.py:911-917): Ritz residual
        |beta_m s_m| <= tol |theta|.  ARPACK checks it only every ncv-1 = 9 products
        and therefore usually overshoots it by far (its Logo estimates agree to
        1e-5); to be as tight, and reproducible to the digits the reference's
        doctest prints, iterations continue -- products are cheap here -- until the
        eigenvalue error estimate resid^2 / (theta_1 - theta_2) is below 1e-5 |theta|
        or ``polish_steps`` products have been spent.
        """
        torch = nat.require_cuda()
        n, L = self.n_vertices, self.L
        if n == 0 or L.nnz == 0:
            return 0.0
        cap = int(min(n, max_steps))
        V = torch.empty(3 * n, dtype=self.dtype, device=self.device)
        scal = torch.zeros(2 * cap + 1 + 4096, dtype=torch.float64, device=self.device)
        done = 0
        theta = None
        converged = False
        while done < cap:
            nxt = min(cap, done + (10 if done == 0 else 5))     # ncv = min(N, 10) first
            self._call("gsp_lanczos", nat.i64(n), nat.i64(L.nnz), L.indptr, L.indices, L.data, V,
                       nat.i32(done), nat.i32(nxt), nat.i32(cap), nat.u64(seed), scal)
            done = nxt
            host = scal.cpu().numpy()
            theta, m, stop, ref_rule = ritz_check(host[:done], host[cap + 1:cap + 1 + done], tol,
                                                  self._sfx == "f32", done >= polish_steps)
            self._lanczos_steps = m
            converged = converged or ref_rule
            if stop:
                return theta
        if converged or cap == n:   # cap == n: the Krylov space is the whole space
            return theta
        raise ValueError("The Lanczos method did not converge. Try to use bounds.")

    def _get_upper_bound(self):
        r"""Algebraic upper bound on the spectrum of L (graph.py:933-960)."""
        if self.lap_type == "normalized":
            return 2
        if self.lap_type != "combinatorial":
            raise ValueError("Unknown Laplacian type {}".format(self.lap_type))
        torch = nat.require_cuda()
        W, Ws, n = self._adjacency, self._symmetric_adjacency(), self.n_vertices
        dw = self._degrees()[0]
        out = torch.empty(5, dtype=torch.float64, device=self.device)
        self._call("gsp_spectral_bounds", nat.i64(n), W.indptr, W.indices, W.data, Ws.indptr,
                   Ws.indices, Ws.data, dw, out)
        max_w, max_dw, max_edge, merris, n_nan = out.cpu().numpy()
        if W.nnz < n * n:                       # np.max of a sparse matrix sees the zeros
            max_w = max(max_w, 0.0)
        bounds = [n * max_w, 2 * max_dw]
        if self.n_edges > 0:
            bounds.append(max_edge)
        bounds.append(float("nan") if n_nan else merris)
        # Python's min() skips a NaN that is not first: with an isolated vertex the
        # reference silently drops the last bound.  Same here.
        return float(min(bounds))


def ritz_check(alpha, beta, tol, single_precision, polish_done):
    """Largest Ritz value of the Lanczos tridiagonal matrix and whether to stop.

    alpha[0..m), beta[0..m): recurrence coefficients so far (beta[j] couples v_j, v_j+1).
    Returns (theta, steps_used, stop).  Stop rule: the reference's (|beta_m s_m| <=
    tol |theta|, graph.py:911-917) and then either the eigenvalue error estimate
    resid^2 / (theta_1 - theta_2) <= 1e-5 |theta| or ``polish_done``; an (almost) zero
    beta_j means an invariant subspace (T_{j+1} exact) and stops at once.
    """
    from scipy.linalg import eigh_tridiagonal
    done = len(alpha)
    scale = max(np.abs(alpha).max(), np.abs(beta).max(), 1e-300)
    floor = (1e-5 if single_precision else 1e-12) * scale
    tiny = np.flatnonzero(beta <= floor)
    m = int(tiny[0]) + 1 if tiny.size else done
    if m == 1:
        theta, second, last = float(alpha[0]), None, 1.0
    else:
        w, v = eigh_tridiagonal(alpha[:m], beta[:m - 1])
        theta, second, last = float(w[-1]), float(w[-2]), abs(float(v[-1, -1]))
    resid = float(beta[m - 1]) * last
    ref_rule = resid <= tol * max(abs(theta), np.finfo(float).eps ** (2.0 / 3))
    gap = max(theta - second, resid) if second is not None else resid
    tight = resid == 0 or resid * resid / max(gap, 1e-300) <= 1e-5 * abs(theta)
    return theta, m, bool(tiny.size or (ref_rule and (tight or polish_done))), ref_rule


def symmetrize_device(W, method="average"):
    """utils.symmetrize(W, method) of a square DeviceCSR, on the device (utils.py:244-277):
    :meth:`DeviceCSR.symmetrize`."""
    return W.symmetrize(method)


def _torch_dtype(torch, dtype):
    if dtype is None:
        return torch.float32
    if isinstance(dtype, torch.dtype):
        out = dtype
    else:
        out = {np.dtype("float32"): torch.float32, np.dtype("float64"): torch.float64}.get(
            np.dtype(dtype))
    if out not in (torch.float32, torch.float64):
        raise TypeError("dtype must be float32 or float64")
    return out
