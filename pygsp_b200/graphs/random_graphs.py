"""Random graph models sampled on the device (csrc/random_graphs.cu, csrc/random_regular.cu).

``ErdosRenyi``, ``BarabasiAlbert`` and ``RandomRegular`` (pygsp/graphs/erdosrenyi.py,
barabasialbert.py, randomregular.py) and the device sampler of
``StochasticBlockModel(backend='device')``.  The draws come from counter-based
Philox streams keyed by a 64-bit key taken from ``np.random.default_rng(seed)``: a graph is a
function of (seed, parameters) alone, whatever the launch shape, and a serial
restatement of the samplers reproduces it bit for bit.  The streams are not the reference's,
so equality with the reference is statistical (DESIGN.md section 4.16).
"""
import ctypes
import math

import numpy as np

from .. import _native as nat
from .csr import DeviceCSR
from .generators import StochasticBlockModel, _device_of
from .graph import Graph, _torch_dtype

# Expected edges per chunk of the SBM walk.  Part of the determinism contract: the graph of a
# key depends on it through the chunk plan.
_CHUNK_TARGET = 64
# Grid cap of the sampling launches (0: the default shape).  Results do not depend on it.
_MAX_BLOCKS = 0
# Pool size below which one CTA finishes a random regular graph by the sequential rule
# (GSPB200_RR_TAIL_STUBS of include/gspb200.h).  Part of the determinism contract.
_TAIL_STUBS = 4096

RECT, TRI_STRICT, TRI_LOOPS, OFF_DIAG = 0, 1, 2, 3
PLAN_COLS = 8


def pair_space(na, nb, same, directed, self_loops):
    """(kind, number of candidate pairs, decoder width) of the block pair (a, b)."""
    if not same:
        return RECT, na * nb, nb
    if directed:
        return (RECT, na * na, na) if self_loops else (OFF_DIAG, na * (na - 1), na)
    return (TRI_LOOPS, na * (na + 1) // 2, na) if self_loops else (TRI_STRICT, na * (na - 1) // 2, na)


def decode_pairs(kind, idx, width):
    """Block-local (i, j) of candidate indices idx (int64 array) -- the decoders of
    csrc/random_graphs.cu, square roots corrected in integers."""
    idx = np.asarray(idx, dtype=np.int64)
    if kind == RECT:
        return idx // width, idx % width
    if kind == OFF_DIAG:
        i, j = idx // (width - 1), idx % (width - 1)
        return i, j + (j >= i)
    s = 1 if kind == TRI_STRICT else -1          # i (i - s) / 2 <= idx < (i + 1) (i + 1 - s) / 2
    i = np.floor((s + np.sqrt(1 + 8 * idx.astype(np.float64))) / 2).astype(np.int64)
    while True:
        lo = i * (i - s) // 2 > idx
        hi = (i + 1) * (i + 1 - s) // 2 <= idx
        if not (lo.any() or hi.any()):
            break
        i = i - lo + hi
    return i, idx - i * (i - s) // 2


def sbm_plan(sizes, M, directed, self_loops, target=None):
    """Chunk plan of the device SBM sampler: (plan (nblk, PLAN_COLS) int64, prob (nblk, 2) float64,
    number of chunks).  Block pairs in (a, b) order, b <= a when undirected (the lower triangle
    of M, as the reference reads it for a sorted z); pairs of probability 0 are left out."""
    target = _CHUNK_TARGET if target is None else target
    k = len(sizes)
    start = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
    plan, prob, cfirst = [], [], 0
    for a in range(k):
        for b in range(k if directed else a + 1):
            kind, n_pairs, width = pair_space(int(sizes[a]), int(sizes[b]), a == b, directed,
                                              self_loops)
            p = float(M[a, b])
            if n_pairs == 0 or p == 0:
                continue
            clen = min(max(math.ceil(target / p), 1), n_pairs)
            plan.append([n_pairs, clen, cfirst, start[a], start[b], width, kind, int(not directed)])
            prob.append([p, math.log1p(-p) if p < 1 else -math.inf])
            cfirst += -(-n_pairs // clen)
    return (np.array(plan, dtype=np.int64).reshape(-1, PLAN_COLS),
            np.array(prob, dtype=np.float64).reshape(-1, 2), cfirst)


def _assemble(rows, cols, N, dt):
    """Unit-weight adjacency of the emitted COO entries; every entry must be distinct."""
    torch = nat.require_cuda()
    W = DeviceCSR.from_coo(rows, cols, torch.ones(rows.numel(), dtype=dt, device=rows.device),
                           (N, N))
    if W.nnz != rows.numel():
        raise nat.NativeError("the sampler emitted %d entries but only %d are distinct"
                              % (rows.numel(), W.nnz))
    return W


def sbm_device(N, k, z, M, directed, self_loops, key, dtype=None, device=None):
    """One SBM adjacency (DeviceCSR, unit weights) drawn on the device with Philox key ``key``.

    z (length N, values in [0, k)) need not be sorted: block-local ids map to vertices through
    its stable sort.  ``ValueError`` when the graph would hold 2^31 entries or more, raised after
    the count pass and before anything is filled."""
    torch = nat.require_cuda()
    dev, dt = _device_of(device), _torch_dtype(torch, dtype)
    z = np.asarray(z, dtype=np.int64)
    plan, prob, n_chunks = sbm_plan(np.bincount(z, minlength=k), M, directed, self_loops)
    with torch.cuda.device(dev):
        perm = torch.sort(torch.from_numpy(z).to(dev), stable=True).indices.int()
        plan_t, prob_t = torch.from_numpy(plan).to(dev), torch.from_numpy(prob).to(dev)
        offsets = torch.empty(n_chunks + 1, dtype=torch.int64, device=dev)
        args = (nat.i64(n_chunks), nat.i64(len(plan)), plan_t, prob_t, nat.u64(key))
        nat.call("gsp_sbm_count", *args, offsets, nat.i32(_MAX_BLOCKS), nat.stream_ptr(dev))
        total = int(offsets[-1].item())
        if total >= 2 ** 31:
            raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                             "supported.".format(total))
        rows = torch.empty(total, dtype=torch.int32, device=dev)
        cols = torch.empty(total, dtype=torch.int32, device=dev)
        nat.call("gsp_sbm_fill", *args, perm, offsets, rows, cols, nat.i32(_MAX_BLOCKS),
                 nat.stream_ptr(dev))
        return _assemble(rows, cols, N, dt)


def barabasi_albert_device(N, m0, m, key, dtype=None, device=None):
    """(adjacency DeviceCSR, rounds) of one Barabasi-Albert graph drawn with Philox key ``key``."""
    torch = nat.require_cuda()
    dev, dt = _device_of(device), _torch_dtype(torch, dtype)
    total = 2 * m * max(N - m0, 0)
    if total >= 2 ** 31:
        raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                         "supported.".format(total))
    rounds = ctypes.c_int(0)
    with torch.cuda.device(dev):
        rows = torch.empty(total, dtype=torch.int32, device=dev)
        cols = torch.empty(total, dtype=torch.int32, device=dev)
        if total:
            nat.call("gsp_barabasi_albert", nat.i64(N), nat.i64(m0), nat.i64(m), nat.u64(key),
                     rows, cols, nat.i32(_MAX_BLOCKS), ctypes.byref(rounds),
                     nat.stream_ptr(dev))
        return _assemble(rows, cols, N, dt), rounds.value


class ErdosRenyi(StochasticBlockModel):
    r"""Erdos Renyi graph (pygsp/graphs/erdosrenyi.py): every edge present with probability p,
    independently, unit weights -- the k = 1 stochastic block model.  ``backend='host'`` takes
    the host sampler of :class:`StochasticBlockModel`."""

    def __init__(self, N=100, p=0.1, directed=False, self_loops=False, connected=False,
                 n_try=10, seed=None, backend="device", **kwargs):
        super().__init__(N=N, k=1, p=p, connected=connected, n_try=n_try, seed=seed,
                         directed=directed, self_loops=self_loops, backend=backend, **kwargs)


class BarabasiAlbert(Graph):
    r"""Barabasi-Albert preferential attachment (pygsp/graphs/barabasialbert.py:43-65).

    The m0 first vertices are disconnected; every later vertex i links to m distinct earlier
    vertices drawn with probability proportional to 1 + degree, as the reference's sequential
    process does.  Sampled on the device in rounds (``gsp_barabasi_albert``); the Philox key is
    ``np.random.default_rng(seed).integers(2**63)``.
    """

    def __init__(self, N=1000, m0=1, m=1, seed=None, **kwargs):
        if m > m0:
            raise ValueError("Parameter m cannot be above parameter m0.")
        self.m0, self.m, self.seed = m0, m, seed
        key = int(np.random.default_rng(seed).integers(2 ** 63))
        W, self._rounds = barabasi_albert_device(N, m0, m, key, kwargs.get("dtype"),
                                                 kwargs.get("device"))
        super().__init__(W, **kwargs)

    def _get_extra_repr(self):
        return dict(m0=self.m0, m=self.m, seed=self.seed)


def random_regular_device(N, k, max_iter, key, dtype=None, device=None):
    """(adjacency DeviceCSR, attempts, rounds) of one random k-regular graph drawn with Philox key
    ``key`` (``gsp_random_regular``).  For k > (N - 1) / 2 the (N - 1 - k)-regular graph is drawn
    and its complement written straight into CSR (``gsp_random_regular_complement``).  The
    arguments must already be valid (see :class:`RandomRegular`)."""
    torch = nat.require_cuda()
    dev, dt = _device_of(device), _torch_dtype(torch, dtype)
    kk = N - 1 - k if 2 * k > N - 1 else k
    attempts, rounds, entries = ctypes.c_int(0), ctypes.c_int(0), ctypes.c_int64(0)
    with torch.cuda.device(dev):
        rows = torch.empty(N * kk, dtype=torch.int32, device=dev)
        cols = torch.empty(N * kk, dtype=torch.int32, device=dev)
        nat.call("gsp_random_regular", nat.i64(N), nat.i64(kk), nat.i32(max_iter), nat.u64(key),
                 rows, cols, nat.i32(_MAX_BLOCKS), ctypes.byref(attempts), ctypes.byref(rounds),
                 ctypes.byref(entries), nat.stream_ptr(dev))
        m = entries.value
        W = _assemble(rows[:m], cols[:m], N, dt)
        if kk != k:
            nnz = N * (N - 1) - W.nnz
            if nnz >= 2 ** 31:
                raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                                 "supported.".format(nnz))
            indptr = torch.empty(N + 1, dtype=torch.int32, device=dev)
            indices = torch.empty(nnz, dtype=torch.int32, device=dev)
            nat.call("gsp_random_regular_complement", nat.i64(N), nat.i64(nnz), W.indptr,
                     W.indices, indptr, indices, nat.stream_ptr(dev))
            W = DeviceCSR(indptr, indices, torch.ones(nnz, dtype=dt, device=dev), (N, N))
        return W, attempts.value, rounds.value


class RandomRegular(Graph):
    r"""Random k-regular graph (pygsp/graphs/randomregular.py): simple, undirected, unit weights,
    every vertex adjacent to exactly k others.

    Stub pairing on the device (``gsp_random_regular``): pairing rounds while more than
    ``_TAIL_STUBS`` stubs are open, then the reference's sequential rule -- draw two open stubs,
    keep the pair if it makes neither a loop nor a repeated edge -- with a restart when no legal
    pair is left, up to ``max_iter`` attempts; the last attempt places its remaining stubs by edge
    switches rather than giving up.  For k > (N - 1) / 2 the complement of an (N - 1 - k)-regular
    graph is built.  The Philox key is ``np.random.default_rng(seed).integers(2**63)``.
    ``_attempts`` and ``_rounds`` record the attempts and pairing rounds used.

    ``ValueError`` when N k is odd (the reference's message), k < 0, k >= N (no such graph),
    max_iter < 1 or N k >= 2^31, before anything is allocated on the device.
    """

    def __init__(self, N=64, k=6, max_iter=10, seed=None, **kwargs):
        self.k = k
        self.max_iter = max_iter
        self.seed = seed
        if (N * k) % 2 == 1:
            raise ValueError("input error: N*d must be even!")
        if k < 0:
            raise ValueError("The degree k must be non-negative, got {}.".format(k))
        if k >= max(N, 1):
            raise ValueError("A {}-regular graph on {} vertices does not exist: k must be below "
                             "N.".format(k, N))
        if max_iter < 1:
            raise ValueError("max_iter must be at least 1, got {}.".format(max_iter))
        if N * k >= 2 ** 31:
            raise ValueError("The graph would have {} entries; at most 2^31 - 1 are "
                             "supported.".format(N * k))
        key = int(np.random.default_rng(seed).integers(2 ** 63))
        W, self._attempts, self._rounds = random_regular_device(
            N, k, max_iter, key, kwargs.get("dtype"), kwargs.get("device"))
        super().__init__(W, **kwargs)
        self.is_regular()

    def is_regular(self):
        r"""Troubleshoot a given regular graph: log the reference's warning when the graph is not
        symmetric, has parallel edges (a weight above 1), is not d-regular or has self-loops.
        Computed on the device from ``is_directed()``, the weights, ``d`` and ``has_loops()``."""
        warn = False
        msg = "The given matrix"
        if self.is_directed():
            warn = True
            msg = "{} is not symmetric,".format(msg)
        if self.W.nnz and bool((self.W.data > 1).any()):
            warn = True
            msg = "{} has parallel edges,".format(msg)
        d = self.d
        if d.size and d.min() != d.max():
            warn = True
            msg = "{} is not d-regular,".format(msg)
        if self.has_loops():
            warn = True
            msg = "{} has self loop.".format(msg)
        if warn:
            self.logger.warning("{}.".format(msg[:-1]))

    def _get_extra_repr(self):
        return dict(k=self.k, seed=self.seed)
