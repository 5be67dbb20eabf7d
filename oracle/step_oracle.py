"""High-precision reference of one fused Chebyshev step, with a per-element error bound.

TEST INFRASTRUCTURE ONLY: nothing under ``pygsp_b200/`` imports this module.

``gsp_cheby_step_*`` (include/gspb200.h) computes, on every row i of its range,

    x_new = alpha * (L x_cur) + beta * x_cur + gamma * x_old          (first: no gamma term)
    r_k   = r_k + ck[k] * x_new        (first: r_k = c0[k]/2 * x_cur + ck[k] * x_new)

or, in the Clenshaw form (``add_source``), x_new = x_new + sum_i cs[i] * s_i with read-only source
blocks s_i and no accumulator.

:func:`step_reference` evaluates the same step in a wider type than the engine's (float64 for
a float32 engine, ``np.longdouble`` for a float64 one) from the engine's own input values and
from the coefficients rounded to the engine type exactly as the kernels round them
(``T(alpha)``, ``T(0.5 * c0)``).  It also returns, for every element, a bound on the distance
between the reference and ANY result produced by the kernels' operation sequence.  A result
outside the bound is wrong: the bound is a proof, not a tuned tolerance.  See
:func:`step_reference` for the derivation.
"""

import numpy as np
from scipy import sparse


def _gamma(k, u):
    """gamma_k = k u / (1 - k u): |prod_{j<=k} (1 + d_j) - 1| <= gamma_k for |d_j| <= u."""
    k = np.asarray(k, dtype=np.float64)
    return k * u / (1.0 - k * u)


def _csr_products(L, x, work):
    """(sum_j w_ij x_j, sum_j |w_ij x_j|) per row and column, in the type ``work``."""
    n = L.shape[0]
    xw = x.astype(work)
    if work == np.float64:            # any summation order: the bound covers every order
        L64 = L.astype(np.float64)
        return np.asarray(L64 @ xw), np.asarray(abs(L64) @ np.abs(xw))
    data = L.data.astype(work)
    S = np.zeros((n, x.shape[1]), dtype=work)
    A = np.zeros((n, x.shape[1]), dtype=work)
    if L.nnz:
        prod = data[:, None] * xw[L.indices]
        rows = np.flatnonzero(np.diff(L.indptr) > 0)
        S[rows] = np.add.reduceat(prod, L.indptr[rows], axis=0)
        A[rows] = np.add.reduceat(np.abs(prod), L.indptr[rows], axis=0)
    return S, A


def step_reference(L, x_cur, x_old, r, alpha, beta, gamma, ck, c0, first, dtype=np.float32,
                   sources=None, cs=None):
    r"""One ``gsp_cheby_step_*`` on all rows of the square CSR ``L`` (values in the engine dtype).

    ``x_cur``, ``x_old``: (n, nsig) in the engine dtype (``x_old`` ignored when ``first``); ``r``:
    (nscales, n, nsig) accumulators before the step (ignored when ``first``); ``ck``, ``c0``: the
    float64 coefficients handed to the library.  Returns ``(x_new, r_new, bound_x, bound_r)``,
    references in the wide type and bounds in float64, shapes (n, nsig) and (nscales, n, nsig).

    ``sources`` (nsrc, n, nsig) in the engine dtype and ``cs`` (nsrc float64 coefficients) model
    the Clenshaw form of the step: after the three operations below, ``x_new = fma(c_i, s_i,
    x_new)`` for i = 0 .. nsrc-1 in that order, and no accumulator (``r`` must be None; r_new and
    bound_r have nscales = 0).  Without ``sources`` the results are those of the plain step.

    Derivation.  u is the engine's unit roundoff (2^-24 float32, 2^-53 float64) and every
    operation of the kernel obeys fl(z) = z (1 + d), |d| <= u, plus an absolute error <= eta
    (half the smallest subnormal) when the result underflows.  gamma_k = k u / (1 - k u), and
    (1 + gamma_j)(1 + gamma_k) <= 1 + gamma_{j+k}.  a, b, g, c, h are alpha, beta, gamma, ck[k]
    and c0[k]/2 rounded to the engine type; they are the exact operands of the kernel.  Row i has
    m stored entries, m' = max(m, 1), and per column

        A = sum_j |w_ij x_j|,   S = sum_j w_ij x_j,   X = a S + b x_c + g x_o   (exact).

    Row sum, ``acc = fma(w_j, x_j, acc)`` in stored order from 0: the j-th product passes
    through m - j + 1 roundings, so |acc - S| <= gamma_m A.

    ``t = b * x_c``, ``x1 = fma(a, acc, t)``, ``x_new = fma(g, x_o, x1)``:

        x_new = (g x_o + (a acc + b x_c (1+d1)) (1+d2)) (1+d3)
        |x_new - X| <= |a| A ((1 + gamma_m)(1+u)^2 - 1) + |b x_c| gamma_3 + |g x_o| gamma_1
                    <= gamma_{m+2} |a| A + gamma_3 |b x_c| + gamma_1 |g x_o|
                    <= gamma_{m'+2} M,        M = |a| A + |b x_c| + |g x_o|  (>= |X|).

    First step (no g term): |x_new - X| <= gamma_{m+1} |a| A + gamma_2 |b x_c| <= gamma_{m'+1} M.

    Accumulator, ``r_new = fma(c, x_new, r_old)`` with R = c X + r_old:

        |r_new - R| <= (1+u) |c| |x_new - X| + u (|c| M + |r_old|)
                    <= gamma_{m'+3} |c| M + gamma_2 |r_old|.

    First step, ``r = fma(c, x_new, h * x_c)`` with R = c X + h x_c:

        |r - R| <= (1+u) |c| |x_new - X| + u |c| M + gamma_2 |h x_c|
                <= gamma_{m'+2} |c| M + gamma_2 |h x_c|.

    Sources (Clenshaw form), c_i = cs[i] rounded to the engine type, Z = sum_i |c_i s_i| and
    x^(0) the x_new above: x^(i+1) = (x^(i) + c_i s_i)(1 + d_i), exact target E = X + sum_i c_i s_i.
    Unrolled, x^(nsrc) = x^(0) prod_i (1 + d_i) + sum_i c_i s_i prod_{j>=i} (1 + d_j), so

        |x^(nsrc) - E| <= (1 + gamma_nsrc) |x^(0) - X| + gamma_nsrc (|X| + Z)
                       <= gamma_{m'+2+nsrc} (M + Z)          (first: gamma_{m'+1+nsrc} (M + Z)),

    using |X| <= M and (1 + gamma_j)(1 + gamma_k) <= 1 + gamma_{j+k}.  Each fma adds at most one
    eta on underflow (the floor counts 2 eta, one smallest subnormal, per source), and the
    reference, one more rounded sum per source, lies within gamma^w_{m'+3+nsrc} (M + Z) of E.

    (The one-rounding terms gamma_1 |r_old| are written gamma_2, which keeps every bound at least
    twice the rounding of the stored result itself, u |R|: the float32 rounding of the exact value
    then sits at most half-way to the bound.  Only these slacks of one u separate the bound
    from the analysis.)

    Underflow: the m + 3 operations of x_new add at most (m |a| + 3) eta, those of r at most
    |c| times that plus 2 eta; the floor below counts 2 eta (one smallest subnormal) for each.

    The reference is itself rounded in the wide type (unit roundoff u_w): it lies within
    gamma^w_{m'+3} M of X and within gamma^w_{m'+5} (|c| M + |r_old| + |h x_c|) of R, which is
    added to the bounds.  So |kernel - reference| <= bound for any kernel that performs exactly
    this operation sequence; the bounds are evaluated in float64 and rounded up by 2^-40.
    """
    dtype = np.dtype(dtype)
    work = np.float64 if dtype == np.float32 else np.longdouble
    u = float(np.finfo(dtype).eps) / 2
    uw = float(np.finfo(work).eps) / 2
    tiny = float(np.finfo(dtype).smallest_subnormal)
    n = L.shape[0]
    x_cur = np.asarray(x_cur, dtype=dtype).reshape(n, -1)
    nsig = x_cur.shape[1]
    ck = np.atleast_1d(np.asarray(ck, dtype=np.float64))
    c0 = np.atleast_1d(np.asarray(c0, dtype=np.float64))
    nscales = 0 if r is None else int(np.asarray(r).shape[0])
    if sources is not None and nscales:
        raise ValueError("the Clenshaw form reads source blocks and writes no accumulator")
    a, b, g = (work(dtype.type(v)) for v in (alpha, beta, gamma))
    cks = [work(dtype.type(ck[k])) for k in range(nscales)]
    hs = [work(dtype.type(0.5 * c0[k])) for k in range(nscales)]

    S, A = _csr_products(L, x_cur, work)
    xc = x_cur.astype(work)
    m = np.diff(L.indptr).astype(np.float64)[:, None]
    mp = np.maximum(m, 1.0)
    x_new = a * S + b * xc
    Mx = np.abs(a) * A + np.abs(b * xc)
    if first:
        gx = _gamma(mp + 1, u)
    else:
        xo = np.asarray(x_old, dtype=dtype).reshape(n, nsig).astype(work)
        x_new = x_new + g * xo
        Mx = Mx + np.abs(g * xo)
        gx = _gamma(mp + 2, u)
    nsrc = 0
    if sources is not None:
        cw = np.atleast_1d(np.asarray(cs, dtype=np.float64)).astype(dtype).astype(work)
        nsrc = len(cw)
        src = np.asarray(sources, dtype=dtype).reshape(nsrc, n, nsig)
        for i in range(nsrc):
            t = cw[i] * src[i].astype(work)
            x_new = x_new + t
            Mx = Mx + np.abs(t)
        gx = _gamma((mp + 1 if first else mp + 2) + nsrc, u)
    Mx64 = Mx.astype(np.float64)
    floor_x = tiny * (m * max(abs(float(a)), 1.0) + 3 + nsrc)
    bound_x = gx * Mx64 + _gamma(mp + 3 + nsrc, uw) * Mx64 + floor_x

    r_new = np.zeros((nscales, n, nsig), dtype=work)
    bound_r = np.zeros((nscales, n, nsig), dtype=np.float64)
    for k in range(nscales):
        c = cks[k]
        if first:
            other = hs[k] * xc
            gc = _gamma(mp + 2, u)
        else:
            other = np.asarray(r[k], dtype=dtype)[:n].astype(work)
            gc = _gamma(mp + 3, u)
        r_new[k] = c * x_new + other
        mo = np.abs(other).astype(np.float64)
        cm = abs(float(c)) * Mx64
        bound_r[k] = (gc * cm + _gamma(2, u) * mo + _gamma(mp + 5, uw) * (cm + mo)
                      + max(abs(float(c)), 1.0) * floor_x + 2 * tiny)
    scale = 1.0 + 2.0 ** -40
    return x_new, r_new, bound_x * scale, bound_r * scale


def mix_reference(sources, c, dtype=np.float32):
    r"""The per-order sources of the wide synthesis, ``u_k = sum_f c'_fk s_f``, with a bound.

    ``sources``: (nsrc, n, nsig) in the engine dtype; ``c``: (nsrc, m) float64 coefficients, of
    which the kernel uses c'_fk = T(c_fk) for k > 0 and T(c_f0 / 2) for k = 0.  Returns ``(u,
    bound)``, shapes (m, n, nsig), the reference in the wide type and the bound in float64.

    Derivation.  The kernel runs ``acc = fma(c'_fk, s_f, acc)`` from acc = 0 in increasing f, so the
    f-th product passes through nsrc - f roundings and, with Z_k = sum_f |c'_fk s_f|,
    |u_k - exact| <= gamma_nsrc Z_k, plus eta per fma on underflow (counted as one smallest
    subnormal per source).  The reference sums the exact products (a product of two engine values
    is exact in the wide type for float32, and within u_w of it for float64) with one rounding
    each, within gamma^w_{nsrc+1} Z_k of the exact sum.  Rounded up by 2^-40 like the step's.
    """
    dtype = np.dtype(dtype)
    work = np.float64 if dtype == np.float32 else np.longdouble
    u = float(np.finfo(dtype).eps) / 2
    uw = float(np.finfo(work).eps) / 2
    tiny = float(np.finfo(dtype).smallest_subnormal)
    c = np.atleast_2d(np.asarray(c, dtype=np.float64)).copy()
    c[:, 0] *= 0.5
    cw = c.astype(dtype).astype(work)
    nsrc, m = c.shape
    src = np.asarray(sources, dtype=dtype)
    shape = src.shape[1:]
    flat = src.reshape(nsrc, -1).astype(work)
    uk = np.zeros((m, flat.shape[1]), dtype=work)
    zk = np.zeros((m, flat.shape[1]), dtype=work)
    for f in range(nsrc):
        uk += cw[f][:, None] * flat[f][None, :]
        zk += np.abs(cw[f][:, None] * flat[f][None, :])
    z = zk.astype(np.float64)
    bound = (float(_gamma(nsrc, u)) + float(_gamma(nsrc + 1, uw))) * z + tiny * nsrc
    return uk.reshape((m,) + shape), bound.reshape((m,) + shape) * (1.0 + 2.0 ** -40)


def violations(got, ref, bound):
    """Boolean mask of the elements where |got - ref| > bound (NaN or Inf in ``got`` counts)."""
    ref = np.asarray(ref)
    diff = np.abs(np.asarray(got).astype(ref.dtype) - ref)
    return ~(diff <= np.asarray(bound, dtype=ref.dtype))


# ------------------------------------------------------------------------ test graphs
def morton_order(points, bits=16):
    """Permutation that sorts 2-D points in [0, 1)^2 along a Z-curve."""
    q = np.minimum((points * (1 << bits)).astype(np.uint64), (1 << bits) - 1)
    code = np.zeros(len(points), dtype=np.uint64)
    for b in range(bits):
        for d in range(2):
            code |= ((q[:, d] >> np.uint64(b)) & np.uint64(1)) << np.uint64(2 * b + d)
    return np.argsort(code, kind="stable")


def sensor_adjacency(n, k=8, seed=0):
    """Random sensor network on the host: n uniform points in the unit square numbered along a
    Z-curve, k-NN graph with Gaussian weights exp(-d^2 / sigma) (sigma = mean neighbour
    distance), symmetrised by averaging -- the construction of ``graphs.Sensor(order='morton')``."""
    from scipy import spatial
    pts = np.random.default_rng(seed).uniform(0, 1, (n, 2))
    pts = pts[morton_order(pts)]
    D, NN = spatial.cKDTree(pts).query(pts, k=k + 1)
    sigma = np.mean(D[:, 1:])
    rows = np.repeat(np.arange(n), k)
    W = sparse.csr_matrix((np.exp(-D[:, 1:].ravel() ** 2 / sigma), (rows, NN[:, 1:].ravel())),
                          shape=(n, n))
    W = ((W + W.T) / 2).tocsr()
    W.sort_indices()
    return W


def scaled_signals(rng, n, nsig, dtype=np.float32):
    """Standard normal rows, column c scaled by 2^((c mod 9) - 4): the scaling is exact, so
    a column or packet permutation changes a value by a factor of at least 2."""
    x = rng.standard_normal((n, nsig))
    x *= 2.0 ** ((np.arange(nsig) % 9) - 4)
    return x.astype(dtype)
