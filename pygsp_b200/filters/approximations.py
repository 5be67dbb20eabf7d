"""Chebyshev approximation of graph filters, device side.

Mirror of ``pygsp/filters/approximations.py``: ``compute_cheby_coeff`` (:9-55,
host quadrature, K+1 scalars per filter), ``cheby_op`` (:58-114, THE hot loop)
and ``cheby_rect`` (:117-163).  The recurrence runs in ``libgspb200``:
one fused CUDA kernel per order (csrc/cheby.cu) instead of SciPy's
``csr_matvecs`` + NumPy temporaries + fancy-indexed accumulation.
"""
import ctypes

import numpy as np

from .. import _native as nat
from .. import utils

_logger = utils.build_logger(__name__)
PATCH_DEFAULT_DTYPE = None     # engine dtype for reference (scipy) graphs, see patch_pygsp()
# filters whose coefficients the fused step takes by value; wider banks and syntheses of more
# features go through the stored basis (cheby_bank_device) and the per-order sources
# (cheby_synthesis_wide_device)
WIDE_BANK = 16


@utils.filterbank_handler
def compute_cheby_coeff(f, m=30, N=None, *args, **kwargs):
    r"""Chebyshev coefficients of filter ``i`` of the bank ``f`` on [0, lmax].

    Chebyshev-Gauss quadrature with ``N`` (default ``m + 1``) nodes:
    ``c[o] = 2/N sum_j g(a cos(t_j) + a) cos(o t_j)``, ``t_j = pi (j + 1/2) / N``,
    ``a = lmax / 2``.  Evaluated on the host in float64: it is K+1 numbers and
    must see exactly the ``G.lmax`` the device recurrence is given.
    """
    G = f.G
    i = kwargs.pop("i", 0)
    if not N:
        N = m + 1
    half = G.lmax / 2.0
    theta = np.pi * (np.arange(N) + 0.5) / N
    samples = f._kernels[i](half * np.cos(theta) + half)
    orders = np.arange(m + 1)[:, None]
    return (2.0 / N) * (np.cos(orders * theta[None, :]) @ samples)


def _as_device_block(G, signal):
    """signal -> contiguous (N, nsig) device tensor in the graph's dtype."""
    torch = nat.require_cuda()
    kind = "cuda"
    if not torch.is_tensor(signal):
        signal = torch.from_numpy(np.ascontiguousarray(np.asarray(signal)))
        kind = "numpy"
    elif not signal.is_cuda:
        kind = "pinned" if signal.is_pinned() else "cpu"
    one_d = signal.dim() == 1
    x = signal.to(device=G.device, dtype=G.dtype, non_blocking=True)
    x = x.reshape(x.shape[0], -1).contiguous()
    return x, one_d, kind


def _is_pinned_block(s, L):
    """A contiguous page-locked host tensor of the engine's dtype, big enough to pipeline."""
    torch = nat.require_cuda()
    return (torch.is_tensor(s) and not s.is_cuda and s.dim() == 2 and s.dtype == L.dtype
            and s.is_contiguous() and s.is_pinned() and s.numel() > 0)


def _leave_device(t, kind):
    torch = nat.require_cuda()
    if kind == "cuda":
        return t
    if kind == "numpy":
        return t.cpu().numpy()
    out = torch.empty(t.shape, dtype=t.dtype, device="cpu", pin_memory=(kind == "pinned"))
    out.copy_(t, non_blocking=False)
    return out


def _laplacian_on_device(G):
    """(DeviceCSR L, lmax) of any graph object offering .L / .lmax / .N.

    A graph of this package already holds L in HBM.  A *reference* pygsp graph
    (scipy ``G.L``) is uploaded once and the copy is cached on the object, so
    that this function can stand in for ``pygsp.filters.approximations.cheby_op``.
    """
    from ..graphs.csr import DeviceCSR
    L = G.L
    if isinstance(L, DeviceCSR):
        return L
    torch = nat.require_cuda()
    cached = getattr(G, "_gspb200_L", None)
    if cached is None or cached[0] is not L:
        dtype = getattr(G, "_gspb200_dtype", None) or PATCH_DEFAULT_DTYPE or torch.float32
        dev = torch.device("cuda:%d" % torch.cuda.current_device())
        cached = (L, DeviceCSR.from_scipy(L, dtype, dev))
        G._gspb200_L = cached
    return cached[1]


def cheby_op_device(L, lmax, c, x, out=None, work=None):
    """Device-to-device core: x (N, nsig) tensor -> r (Nscales, N, nsig) tensor.

    ``out`` / ``work`` ((Nscales, N, nsig) and (2, N, nsig), contiguous) may be given by callers
    that keep their buffers (the column-chunk pipeline of host signals)."""
    torch = nat.require_cuda()
    c = np.atleast_2d(np.asarray(c, dtype=np.float64))
    nscales, M = c.shape
    if M < 2:
        raise TypeError("The coefficients have an invalid shape")
    n, nsig = x.shape
    c = np.ascontiguousarray(c)
    r = out if out is not None else torch.empty((nscales, n, nsig), dtype=L.dtype, device=L.device)
    if work is None:
        work = torch.empty((2, n, nsig), dtype=L.dtype, device=L.device)
    plan = L.tile_plan(nsig, nscales)
    with torch.cuda.device(L.device):
        nat.call("gsp_cheby_op_" + nat.suffix(L.dtype), nat.i64(n), nat.i64(L.nnz), L.indptr,
                 L.indices, L.data, nat.f64(lmax), c, nat.i32(nscales), nat.i32(M), x,
                 nat.i64(nsig), r, work, plan, nat.stream_ptr(L.device))
    return r


def _free_device_bytes(device):
    torch = nat.require_cuda()
    free, _ = torch.cuda.mem_get_info(device)
    return free + torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device)


def cheby_bank_device(L, lmax, c, x, max_columns=None):
    """Any filter bank through a stored Chebyshev basis: x (N, nsig) tensor -> (Nf, N, nsig).

    The recurrence writes T_k x (k < m) into a basis buffer with no accumulator, and one combine
    pass forms every r_i = sum_k c_ik T_k x (csrc/cheby_bank.cu, ``gsp_cheby_op_basis_*``): the
    basis is read once and each output written once, however many filters there are.  The result
    is the bits of :func:`cheby_op_device` on the same bank.  The basis takes m N nsig elements;
    when that does not fit in the device memory left once the output is allocated (or
    ``max_columns`` is given) the columns are processed in chunks, with the same bits, since no
    sum mixes columns."""
    torch = nat.require_cuda()
    c = np.ascontiguousarray(np.atleast_2d(np.asarray(c, dtype=np.float64)))
    nf, m = c.shape
    if m < 2:
        raise TypeError("The coefficients have an invalid shape")
    n, nsig = x.shape
    out = torch.empty((nf, n, nsig), dtype=L.dtype, device=L.device)
    if nsig == 0 or n == 0:
        return out
    item = x.element_size()
    per_column = m * n * item
    if max_columns is None:
        free = _free_device_bytes(L.device)
        max_columns = int(free * 0.9) // per_column
        if max_columns < 1:
            raise ValueError(
                "The Chebyshev basis of one signal ({0} vectors of {1} x {2} bytes, {3:.2f} GB) "
                "does not fit in the free device memory ({4:.2f} GB). Lower the order.".format(
                    m, n, item, per_column / 2 ** 30, free / 2 ** 30))
    step = max(1, min(int(max_columns), nsig))
    cd = torch.as_tensor(c, device=L.device)
    basis = torch.empty((m, n, step), dtype=L.dtype, device=L.device)
    with torch.cuda.device(L.device):
        for j0 in range(0, nsig, step):
            j1 = min(nsig, j0 + step)
            b = j1 - j0
            if b == nsig:
                buf, xc = basis, x
            else:
                # the chunk is staged in slot 0 of the basis, where the recurrence reads T_0
                buf = basis.view(-1)[:m * n * b].view(m, n, b)
                buf[0].copy_(x[:, j0:j1])
                xc = buf[0]
            nat.call("gsp_cheby_op_basis_" + nat.suffix(L.dtype), nat.i64(n), nat.i64(L.nnz),
                     L.indptr, L.indices, L.data, nat.f64(lmax), cd, nat.i32(nf), nat.i32(m), xc,
                     nat.i64(b), buf, out[:, :, j0:], nat.i64(nsig), L.tile_plan(b, 0),
                     nat.stream_ptr(L.device))
    return out


def cheby_synthesis_wide_device(L, lmax, c, sources):
    """sum_f p_f(L) s_f for any number of source blocks, device to device: (N, nsig).

    ``sources`` is (nsrc, N, nsig), ``c`` (nsrc, M).  One mix pass forms the per-order sources
    u_k = sum_f c_fk s_f (c_f0 halved) and ONE Clenshaw recurrence runs with the source of order k
    (csrc/cheby_bank.cu, ``gsp_cheby_synthesis_wide_*``): K SpMMs, where the reference's synthesis
    runs nsrc forward recurrences (filter.py:313-322).  Same value as
    :func:`cheby_clenshaw_device`, different rounding.  Work memory: (M + 2) N nsig elements."""
    torch = nat.require_cuda()
    c = np.ascontiguousarray(np.atleast_2d(np.asarray(c, dtype=np.float64)))
    nsrc, m = c.shape
    if m < 2:
        raise TypeError("The coefficients have an invalid shape")
    if sources.dim() == 2:
        sources = sources[None]
    if sources.shape[0] != nsrc:
        raise ValueError("one coefficient row per source block")
    sources = sources.contiguous()
    _, n, nsig = sources.shape
    out = torch.empty((n, nsig), dtype=L.dtype, device=L.device)
    if n == 0 or nsig == 0:
        return out
    work = torch.empty((m + 2, n, nsig), dtype=L.dtype, device=L.device)
    cd = torch.as_tensor(c, device=L.device)
    with torch.cuda.device(L.device):
        nat.call("gsp_cheby_synthesis_wide_" + nat.suffix(L.dtype), nat.i64(n), nat.i64(L.nnz),
                 L.indptr, L.indices, L.data, nat.f64(lmax), cd, nat.i32(nsrc), nat.i32(m),
                 sources, nat.i64(nsig), out, work, L.tile_plan(nsig, 1), nat.stream_ptr(L.device))
    return out


def cheby_clenshaw_device(L, lmax, c, sources, out=None, work=None):
    """sum_i p_i(L) s_i by ONE backward (Clenshaw) recurrence, device to device.

    ``sources``: (nsrc, N, nsig) tensor (or (N, nsig) for a single filter), ``c``:
    (nsrc, M) coefficients.  With one source this is the single-filter filtering of
    :func:`cheby_op_device` at 4 instead of 5 passes over the signal block per order; with
    nsrc = Nf sources it is the *synthesis* of ``Filter.filter`` in K SpMMs instead of the
    reference's Nf * K (filter.py:313-322), because Clenshaw's recurrence is linear in its
    source term: b_k = sum_i c_ik s_i + 2 Lt b_{k+1} - b_{k+2}  (SURVEY.md 8f).
    Returns (N, nsig).  ``work`` is (2, N, nsig); with (3, N, nsig), or none, a single float32
    source on a block larger than L2 runs its middle steps two per launch (same bits).
    """
    torch = nat.require_cuda()
    c = np.ascontiguousarray(np.atleast_2d(np.asarray(c, dtype=np.float64)))
    if c.shape[1] < 2:
        raise TypeError("The coefficients have an invalid shape")
    if sources.dim() == 2:
        sources = sources[None]
    nsrc, n, nsig = sources.shape
    if nsrc != c.shape[0]:
        raise ValueError("one coefficient row per source block")
    if nsrc > 16:
        raise ValueError("at most 16 source blocks per call")
    sources = sources.contiguous()
    if out is None:
        out = torch.empty((n, nsig), dtype=L.dtype, device=L.device)
    plan = L.tile_plan(nsig, nsrc)
    if nsrc == 1 and plan is not None:
        # one float32 source: the tiled steps gather from each tile's neighbour ring in shared
        # memory where the rings fit, and on a block larger than L2 the middle steps run two per
        # launch, which takes a third work block (a caller's two-block work keeps single steps)
        ring = L.ring_plan(plan.rows_per_tile)
        if ring is not None and not nat.lib().gsp_cheby_ring_fits(
                ring.ring_max, nat.i64(nsig), ctypes.byref(plan)):
            ring = None
        tables, tile_done = (None,) * 4, None
        if ((work is None or work.shape[0] >= 3)
                and nat.lib().gsp_cheby_clenshaw_pairs_wanted(nat.i64(n), nat.i64(nsig),
                                                              ctypes.byref(plan))):
            tables = L.pair_plan(plan.rows_per_tile)
            tile_done = torch.empty(n // plan.rows_per_tile, dtype=torch.int32, device=L.device)
        if work is None:
            work = torch.empty((2 if tile_done is None else 3, n, nsig), dtype=L.dtype,
                               device=L.device)
        with torch.cuda.device(L.device):
            nat.call("gsp_cheby_clenshaw_ring_f32", nat.i64(n), nat.i64(L.nnz), L.indptr,
                     L.indices, L.data, nat.f64(lmax), c, nat.i32(1), nat.i32(c.shape[1]),
                     sources, nat.i64(nsig), out, work, plan, ring, *tables, tile_done,
                     nat.stream_ptr(L.device))
        return out
    if work is None:
        work = torch.empty((2, n, nsig), dtype=L.dtype, device=L.device)
    with torch.cuda.device(L.device):
        nat.call("gsp_cheby_clenshaw_" + nat.suffix(L.dtype), nat.i64(n), nat.i64(L.nnz),
                 L.indptr, L.indices, L.data, nat.f64(lmax), c, nat.i32(nsrc),
                 nat.i32(c.shape[1]), sources, nat.i64(nsig), out, work, plan,
                 nat.stream_ptr(L.device))
    return out


def cheby_op(G, c, signal, **kwargs):
    r"""Chebyshev polynomial of the graph Laplacian applied to a signal block.

    Same contract as the reference (approximations.py:58-114): ``c`` is one
    coefficient vector or an (Nscales, M) array / list of vectors, ``signal``
    is (N,) or (N, Nsig); the result is (Nscales*N,) or (Nscales*N, Nsig) with
    filter-major row blocks.  ``M < 2`` raises TypeError.  NumPy in -> NumPy
    out, CUDA tensor in -> CUDA tensor out.  The arithmetic type is the
    graph's (float32 by default; the reference always computes in float64).
    A single filter is evaluated by Clenshaw's backward recurrence (one pass less over the
    signal block per order, same value, different rounding); ``clenshaw=False`` keeps the
    reference's forward recurrence and operation order.
    """
    if not isinstance(c, np.ndarray):
        c = np.array(c)
    c = np.atleast_2d(c)
    if c.shape[1] < 2:
        raise TypeError("The coefficients have an invalid shape")
    L = _laplacian_on_device(G)
    x, one_d, kind = _as_device_block(_GraphView(L), signal)
    if x.shape[0] != G.N:
        raise ValueError("First dimension must be the number of vertices "
                         "G.N = {}, got {}.".format(G.N, tuple(x.shape)))
    clenshaw = kwargs.get("clenshaw", None)
    if clenshaw and c.shape[0] != 1:
        raise ValueError("clenshaw=True evaluates a single filter")
    if clenshaw is None:
        clenshaw = c.shape[0] == 1
    if clenshaw:
        r = cheby_clenshaw_device(L, G.lmax, c[0], x)
    elif c.shape[0] > WIDE_BANK:
        r = cheby_bank_device(L, G.lmax, c, x)
    else:
        r = cheby_op_device(L, G.lmax, c, x)
    r = r.reshape(c.shape[0] * G.N, x.shape[1])
    if one_d:
        r = r.reshape(-1)
    out = _leave_device(r, kind)
    if kind == "numpy" and not isinstance(G.L, type(L)):
        out = out.astype(np.float64, copy=False)     # a reference graph expects float64 back
    return out


class _GraphView:
    def __init__(self, L):
        self.device, self.dtype = L.device, L.dtype


def cheby_rect(G, bounds, signal, **kwargs):
    r"""Ideal band-pass [bounds[0], bounds[1]] by closed-form Chebyshev coefficients.

    Reference: approximations.py:117-163.  The expansion coefficients of the
    rectangle are c_0/2 = (b1-b2)/pi, c_k = 2/(k pi) (sin k b1 - sin k b2) with
    b = arccos(2 bounds / lmax - 1); the recurrence is the one of ``cheby_op``,
    so the same fused kernel is used with these coefficients.
    """
    if not (isinstance(bounds, (list, np.ndarray)) and len(bounds) == 2):
        raise ValueError("Bounds of wrong shape.")
    bounds = np.array(bounds, dtype=np.float64)
    order = int(kwargs.pop("order", 30))
    b1, b2 = np.arccos(2.0 * bounds / G.lmax - 1.0)
    k = np.arange(1, order + 1)
    c = np.empty(order + 1)
    c[0] = 2.0 * (b1 - b2) / np.pi
    c[1:] = 2.0 / (k * np.pi) * (np.sin(k * b1) - np.sin(k * b2))
    return cheby_op(G, c, signal)


def compute_jackson_cheby_coeff(filter_bounds, delta_lambda, m):
    r"""Chebyshev and Jackson-damped coefficients of an ideal band-pass.

    Reference: approximations.py:166-225.  For the band [a, b] inside
    [lambda_min, lambda_max], mapped to [-1, 1]: ``ch[0] = 2/pi (acos a' - acos b')``,
    ``ch[i] = 2/(pi i) (sin(i acos a') - sin(i acos b'))``; the Jackson factors
    ``g_i = ((1 - i/(m+2)) sin(t) cos(i t) + cos(t) sin(i t)/(m+2)) / sin(t)``,
    ``t = pi/(m+2)``, damp the Gibbs oscillations.  Returns ``(ch, ch * g)``; either
    feeds :func:`cheby_op` directly (host code, m+1 numbers).  Unlike the reference
    the caller's ``filter_bounds`` list is not modified.
    """
    lo, hi = float(delta_lambda[0]), float(delta_lambda[1])
    a, b = float(filter_bounds[0]), float(filter_bounds[1])
    if lo > a or hi < b:
        raise ValueError("Bounds of the filter are out of the lambda values")
    if lo > hi:
        raise ValueError("lambda_min is greater than lambda_max")
    half, mid = (hi - lo) / 2, (hi + lo) / 2
    ta, tb = np.arccos((a - mid) / half), np.arccos((b - mid) / half)
    i = np.arange(1, m + 1)
    ch = np.empty(m + 1)
    ch[0] = 2 / np.pi * (ta - tb)
    ch[1:] = 2 / (np.pi * i) * (np.sin(i * ta) - np.sin(i * tb))
    j = np.arange(m + 1)
    t = np.pi / (m + 2)
    damp = ((1 - j / (m + 2)) * np.sin(t) * np.cos(j * t) + np.cos(t) * np.sin(j * t) / (m + 2)) / np.sin(t)
    return ch, ch * damp


# ------------------------------------------------------------------- diagonal moments
def cheby_square_coeff(c):
    r"""Chebyshev series of ``p^2`` for ``p = c[0]/2 T_0 + sum_k c[k] T_k`` (the reference's
    convention, approximations.py:99-112), in the same convention: ``p^2 = d[0]/2 T_0 +
    sum_n d[n] T_n``, ``n <= 2 (len(c) - 1)``.  From ``T_j T_k = (T_{j+k} + T_{|j-k|}) / 2``.
    ``c`` (m + 1,) gives (2m + 1,); an (Nf, m + 1) array gives (Nf, 2m + 1).  Host, float64."""
    c = np.asarray(c, dtype=np.float64)
    one = c.ndim == 1
    c = np.atleast_2d(c)
    nf, K = c.shape
    a = c.copy()
    a[:, 0] *= 0.5                                  # plain coefficients of T_0 .. T_m
    e = np.zeros((nf, 2 * K - 1))
    for j in range(K):
        # a_j a_k / 2 goes to T_{j+k} and to T_{|j-k|}
        e[:, j:j + K] += 0.5 * a[:, j:j + 1] * a
        diff = np.abs(j - np.arange(K))
        np.add.at(e, (slice(None), diff), 0.5 * a[:, j:j + 1] * a)
    e[:, 0] *= 2.0                                  # back to the c0/2 convention
    return e[0] if one else e


def cheby_moments_device(L, lmax, order, width=None):
    r"""Diagonal Chebyshev moments ``mu[i, n] = (T_n(Lt))_ii``, ``Lt = 2 L / lmax - I``,
    n = 0 .. 2 order: a device (N, 2 order + 1) float64 tensor.

    For every probe block of ``width`` identity columns (csrc/moments.cu), ``order`` steps of
    the Chebyshev recurrence (``gsp_cheby_step_*`` with no accumulator: the tiled kernel at
    float32 widths 8-128) give T_1 .. T_order of the block, and after each step one pass sums
    ``||T_{k+1} e_i||^2`` and ``<T_{k+1} e_i, T_k e_i>`` in float64; ``mu_{2k} = 2 ||T_k e_i||^2 - 1``
    and ``mu_{2k+1} = 2 <T_{k+1} e_i, T_k e_i> - mu_1``.  Then ``||p(L) e_i||^2 = mu[i] . d`` with
    d of :func:`cheby_square_coeff` (d[0] halved) for any p of degree <= order.  A vertex's row is
    the same bits whatever the width or the block it falls in.  The default width is 128 columns
    for float32 and 64 for float64; it is lowered when two (N, width) blocks do not fit in the
    free device memory left once mu is allocated."""
    torch = nat.require_cuda()
    order = int(order)
    if order < 1:
        raise ValueError("The order must be at least 1, got {}.".format(order))
    n = L.shape[0]
    if L.shape[1] != n:
        raise ValueError("The Laplacian must be square, got shape {}.".format(tuple(L.shape)))
    dev, sfx = L.device, nat.suffix(L.dtype)
    item = L.data.element_size()
    if width is None:
        width = 128 if L.dtype == torch.float32 else 64
    width = max(1, min(int(width), n))
    K = 2 * order + 1
    free, _ = torch.cuda.mem_get_info(dev)
    free += torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    mu_bytes = n * K * 8
    # two probe blocks, the step sums and the reduction partials per column
    per_column = 2 * n * item + order * 2 * 8 + 264 * 2 * 8
    room = int(free * 0.9) - mu_bytes
    if room < per_column:
        raise ValueError(
            "The moments (N = {0}, order {1}: {2:.2f} GB) and one probe column do not fit in the "
            "free device memory ({3:.2f} GB). Lower the order.".format(
                n, order, mu_bytes / 2 ** 30, free / 2 ** 30))
    width = min(width, room // per_column)
    mu = torch.empty((n, K), dtype=torch.float64, device=dev)
    blocks = torch.empty((2, n, width), dtype=L.dtype, device=dev)
    sums = torch.empty((order, 2, width), dtype=torch.float64, device=dev)
    zero = np.zeros(1)
    stream = nat.stream_ptr(dev)
    with torch.cuda.device(dev):
        for v0 in range(0, n, width):
            b = min(width, n - v0)
            A = blocks[0].view(-1)[:n * b].view(n, b)       # T_{k-1}, then T_{k+1}
            B = blocks[1].view(-1)[:n * b].view(n, b)       # T_k
            plan = L.tile_plan(b, 0)
            nat.call("gsp_probe_block_" + sfx, nat.i64(n), nat.i64(v0), nat.i64(b), A, stream)
            # T_1 = (2 / lmax) L T_0 - T_0
            nat.call("gsp_cheby_step_" + sfx, nat.i32(1), nat.i64(0), nat.i64(n), nat.i64(L.nnz),
                     L.indptr, L.indices, L.data, A, A, B, B, nat.i64(n), nat.i64(b), nat.i32(0),
                     zero, zero, nat.f64(2.0 / lmax), nat.f64(-1.0), nat.f64(0.0), plan, stream)
            nat.call("gsp_cheby_moments_step_" + sfx, nat.i64(n), B, A, nat.i64(b),
                     nat.i32(order), nat.i32(0), sums, stream)
            cur, old = B, A
            for k in range(1, order):
                # T_{k+1} = (4 / lmax) L T_k - 2 T_k - T_{k-1}, written over T_{k-1} (row-local)
                nat.call("gsp_cheby_step_" + sfx, nat.i32(0), nat.i64(0), nat.i64(n),
                         nat.i64(L.nnz), L.indptr, L.indices, L.data, cur, old, old, old,
                         nat.i64(n), nat.i64(b), nat.i32(0), zero, zero, nat.f64(4.0 / lmax),
                         nat.f64(-2.0), nat.f64(-1.0), plan, stream)
                nat.call("gsp_cheby_moments_step_" + sfx, nat.i64(n), old, cur, nat.i64(b),
                         nat.i32(order), nat.i32(k), sums, stream)
                cur, old = old, cur
            nat.call("gsp_cheby_moments_finish", nat.i64(n), nat.i32(order), nat.i64(v0),
                     nat.i64(b), sums, mu, stream)
    return mu


# ------------------------------------------------------------------------------ Lanczos
def _check_square(shape):
    """Lanczos needs a square matrix: its products are read back as basis vectors."""
    if len(shape) != 2 or shape[0] != shape[1]:
        raise ValueError("The matrix must be square, got shape {}.".format(tuple(shape)))


def _krylov_basis(L, x, order):
    """One Lanczos process per column of the device block x (N, nsig), csrc/krylov.cu.

    Returns the device basis (order + 1, N, nsig) (slot ``order`` is workspace) and, on the
    host, alpha and beta (order, nsig), V^T x (order, nsig) and the Krylov dimensions m (nsig,):
    the only transfer, O(order * nsig) numbers."""
    torch = nat.require_cuda()
    n, nsig = x.shape
    _check_square(L.shape)
    V = torch.empty((order + 1, n, nsig), dtype=L.dtype, device=L.device)
    small = torch.empty((3, order, nsig), dtype=torch.float64, device=L.device)
    m = torch.empty(nsig, dtype=torch.int32, device=L.device)
    with torch.cuda.device(L.device):
        nat.call("gsp_krylov_basis_" + nat.suffix(L.dtype), nat.i64(n), nat.i64(L.shape[1]),
                 L.indptr, L.indices, L.data, x, nat.i64(nsig), nat.i32(order), V, small[0], small[1], small[2], m,
                 nat.stream_ptr(L.device))
    small, m = small.cpu().numpy(), m.cpu().numpy()
    return V, small[0], small[1], small[2], m


def _tridiagonals(alpha, beta):
    """T_j (order x order) of every column: (nsig, order, order)."""
    order, nsig = alpha.shape
    T = np.zeros((nsig, order, order))
    i = np.arange(order)
    T[:, i, i] = alpha.T
    T[:, i[1:], i[:-1]] = T[:, i[:-1], i[1:]] = beta[1:].T
    return T


def _lanczos_coefficients(evaluate, alpha, beta, vs, m):
    """W (Nf, order, nsig): column j's combination Q_j f(max(Theta_j, 0)) Q_j^T (V_j^T s_j)
    over its leading m_j x m_j block, zero past it.  Host float64 ``eigh``, batched over the
    columns of one Krylov dimension."""
    order, nsig = alpha.shape
    T = _tridiagonals(alpha, beta)
    W = None
    for mj in np.unique(m[m > 0]):
        cols = np.flatnonzero(m == mj)
        e, Q = np.linalg.eigh(T[np.ix_(cols, np.arange(mj), np.arange(mj))])   # (c, m), (c, m, m)
        e[e < 0] = 0
        fe = np.asarray(evaluate(e), dtype=np.float64).reshape(-1, cols.size, mj)
        if W is None:
            W = np.zeros((fe.shape[0], order, nsig))
        proj = np.einsum("cki,ck->ci", Q, vs[:mj, cols].T)
        W[:, :mj, cols] = np.einsum("cik,fck->fic", Q, fe * proj[None])
    if W is None:                                     # every column is zero
        W = np.zeros((np.asarray(evaluate(np.zeros(1))).reshape(-1, 1).shape[0], order, nsig))
    return W


def lanczos_op_device(L, evaluate, x, order, max_columns=None):
    """Device-to-device core of :func:`lanczos_op`: x (N, nsig) tensor -> (Nf, N, nsig) tensor.

    The basis takes (order + 1) N nsig elements.  When that does not fit in the device memory
    left once the output is allocated (or ``max_columns`` is given) the columns are processed in
    chunks; the results are the same bits, since no sum mixes columns or depends on their
    number."""
    torch = nat.require_cuda()
    n, nsig = x.shape
    nf = np.asarray(evaluate(np.zeros(1))).reshape(-1, 1).shape[0]
    out = torch.empty((nf, n, nsig), dtype=L.dtype, device=L.device)
    if nsig == 0:
        return out
    item = x.element_size()
    # basis, the column's copy of the signal when chunked, reduction partials, W
    per_column = (order + 2) * n * item + 264 * order * 8 + nf * order * 8
    if max_columns is None:
        free, _ = torch.cuda.mem_get_info(L.device)
        free += torch.cuda.memory_reserved(L.device) - torch.cuda.memory_allocated(L.device)
        max_columns = int(free * 0.9) // per_column
        if max_columns < 1:
            raise ValueError(
                "The Lanczos basis of one signal ({0} vectors of {1} x {2} bytes, {3:.2f} GB) does "
                "not fit in the free device memory ({4:.2f} GB). Lower the order.".format(
                    order + 1, n, item, per_column / 2 ** 30, free / 2 ** 30))
    step = max(1, min(int(max_columns), nsig))
    for j0 in range(0, nsig, step):
        j1 = min(nsig, j0 + step)
        xc = x if (j0, j1) == (0, nsig) else x[:, j0:j1].contiguous()
        V, alpha, beta, vs, m = _krylov_basis(L, xc, order)
        W = _lanczos_coefficients(evaluate, alpha, beta, vs, m)
        Wd = torch.as_tensor(W, device=L.device).contiguous()
        with torch.cuda.device(L.device):
            nat.call("gsp_krylov_combine_" + nat.suffix(L.dtype), nat.i64(n), V, nat.i64(order),
                     Wd, nat.i64(nf), nat.i64(j1 - j0), out[:, :, j0:], nat.i64(nsig),
                     nat.stream_ptr(L.device))
        del V
    return out


def lanczos_op(f, s, order=30):
    r"""Lanczos approximation of the filter bank ``f`` applied to ``s``.

    Same contract as the reference (approximations.py:228-278): ``s`` (N,) gives (Nf*N,), ``s``
    (N, Nv) gives (Nf*N, Nv), with filter-major row blocks as in :func:`cheby_op`.  Column j is
    ``V_j Q_j f(max(Theta_j, 0)) Q_j^T (V_j^T s_j)`` where ``V_j`` is the order-``order`` Krylov
    basis of L and s_j (full reorthogonalisation) and ``Q_j Theta_j Q_j^T`` the eigendecomposition
    of its tridiagonal ``T_j``.  Each column has its own process on the device (csrc/krylov.cu);
    the ``eigh`` of the small ``T_j`` runs on the host in float64.  A column whose Krylov space
    becomes invariant stops growing (the result is then exact) and a zero column gives zeros; the
    reference fails on both.  Input and output kinds and the arithmetic type follow
    :func:`cheby_op`.
    """
    order = int(order)
    if order < 1:
        raise ValueError("The order must be at least 1, got {}.".format(order))
    G = f.G
    L = _laplacian_on_device(G)
    x, one_d, kind = _as_device_block(_GraphView(L), s)
    if x.shape[0] != G.N:
        raise ValueError("First dimension must be the number of vertices "
                         "G.N = {}, got {}.".format(G.N, tuple(x.shape)))
    r = lanczos_op_device(L, f.evaluate, x, order)
    r = r.reshape(r.shape[0] * G.N, x.shape[1])
    if one_d:
        r = r.reshape(-1)
    out = _leave_device(r, kind)
    if kind == "numpy" and not isinstance(G.L, type(L)):
        out = out.astype(np.float64, copy=False)     # a reference graph expects float64 back
    return out


def _orth_from_gram(C, M, order, m):
    """The reference's ``||V^T V - M||_F`` after each step (approximations.py:314, 337) from the
    Gram C of the final basis: vector i of signal j is in place after step k when
    i <= min(k, m_j - 1), and a vector not yet in place is zero, so each of its entries of
    V^T V - M is -M."""
    total = M * order
    orth = np.zeros(order)
    for k in range(order):
        idx = np.concatenate([j * order + np.arange(min(k + 1, int(m[j]))) for j in range(M)])
        sub = C[np.ix_(idx, idx)] - M
        orth[k] = np.sqrt(np.sum(sub ** 2) + (total ** 2 - idx.size ** 2) * float(M) ** 2)
    return orth


def lanczos(A, order, x):
    r"""Lanczos bases of ``A`` for the columns of ``x`` (approximations.py:281-341).

    ``A`` is a :class:`~pygsp_b200.graphs.csr.DeviceCSR` or a SciPy sparse / dense NumPy matrix
    (uploaded as float64 CSR); ``x`` is (N,) or (N, M).  Returns ``(V, H, orth)`` in the
    reference's layout: V (N, M*order) with signal j's k-th vector in column ``j*order + k``, in
    the kind of ``x``; H (order, M*order) with signal j's tridiagonal T_j in columns
    ``j*order .. j*order + order - 1``; orth[k] = ``||V^T V - M||_F`` over the basis as it
    stands after step k.  The M processes are independent (the reference couples them and
    returns the first signal's T only; for M = 1 the two agree).  A signal whose Krylov space
    becomes invariant after m < order steps keeps zero vectors and a zero T past m.
    """
    from scipy import sparse
    from ..graphs.csr import DeviceCSR
    from ..graphs.fourier import block_gram
    order = int(order)
    if order < 1:
        raise ValueError("The order must be at least 1, got {}.".format(order))
    _check_square(A.shape if hasattr(A, "shape") else np.shape(A))
    torch = nat.require_cuda()
    if not isinstance(A, DeviceCSR):
        dev = torch.device("cuda:%d" % torch.cuda.current_device())
        A = DeviceCSR.from_scipy(sparse.csr_matrix(A), torch.float64, dev)
    x, _, kind = _as_device_block(_GraphView(A), x)
    n, M = x.shape
    if n != A.shape[0]:
        raise ValueError("x has {} rows, A is {} x {}.".format(n, *A.shape))
    if M == 0:
        return _leave_device(x[:, :0], kind), np.zeros((order, 0)), np.zeros(order)
    Vb, alpha, beta, _, m = _krylov_basis(A, x, order)
    V = Vb[:order].permute(1, 2, 0).reshape(n, M * order).contiguous()
    del Vb
    C = block_gram(V, V).cpu().numpy()
    T = _tridiagonals(alpha, beta)
    H = np.concatenate(list(T), axis=1)
    return _leave_device(V, kind), H, _orth_from_gram(C, M, order, m)
