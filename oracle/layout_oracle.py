"""Float64 restatement of the reference's Fruchterman-Reingold layout, with a per-element bound
on one step.

TEST INFRASTRUCTURE ONLY: nothing under ``pygsp_b200/`` imports this module.

:func:`step` and :func:`run` restate ``_sparse_fruchterman_reingold``
(pygsp/graphs/_layout.py:169-219) in the reference's own operation order and array shapes,
so they reproduce its results bit for bit; the binary adjacency ``A = W > 0`` (graph.py:718) is
read row by row from a SciPy CSR ``W`` instead of a LIL matrix.  :func:`fruchterman_reingold`
adds the argument handling and rescale of ``_fruchterman_reingold`` (:121-166, :222-233).

:func:`step_bound` bounds the distance between this step and ANY evaluation of the same step
that sums the same terms in another order (the device's, csrc/layout.cu).  The iteration is
chaotic -- a rounding difference grows by orders of magnitude over 50 iterations -- so the
device is held to the reference one step at a time, from the same state.
"""
import numpy as np
from scipy import sparse

U = np.finfo(np.float64).eps / 2     # unit roundoff of float64


def _adjacency_row(W, i):
    """A[i, :].toarray() of A = W > 0: a (1, N) boolean row (_layout.py:207)."""
    row = np.zeros((1, W.shape[0]), dtype=bool)
    s, e = W.indptr[i], W.indptr[i + 1]
    row[0, W.indices[s:e][W.data[s:e] > 0]] = True
    return row


def displacement(pos, W, k, i):
    """The force on vertex i (_layout.py:200-211), shape (dim,)."""
    delta = (pos[i] - pos).T
    distance = np.sqrt((delta ** 2).sum(axis=0))
    distance = np.where(distance < 0.01, 0.01, distance)
    Ai = _adjacency_row(W, i)
    return (delta * (k * k / distance ** 2 - Ai * distance / k)).sum(axis=1)


def _move(pos, displacement, t):
    """The update of _layout.py:212-215 on the columns given (returns the new positions)."""
    length = np.sqrt((displacement ** 2).sum(axis=0))
    length = np.where(length < 0.01, 0.1, length)
    return pos + (displacement * t / length).T


def step(pos, W, k, t, fixed=(), rows=None):
    """One iteration at temperature t (_layout.py:195-215).  Returns the new positions of
    ``rows`` (all by default), shape (len(rows), dim)."""
    W = sparse.csr_matrix(W)
    rows = np.arange(pos.shape[0]) if rows is None else np.asarray(rows)
    fixed = list(fixed)
    disp = np.zeros((pos.shape[1], len(rows)))
    for c, i in enumerate(rows):
        if i in fixed:
            continue
        disp[:, c] += displacement(pos, W, k, i)
    return _move(pos[rows], disp, t)


def run(W, dim, k, pos, fixed, iterations, seed):
    """``_sparse_fruchterman_reingold`` (_layout.py:169-219); ``pos`` is updated in place."""
    W = sparse.csr_matrix(W)
    nnodes = W.shape[0]
    if pos is None:
        pos = np.random.default_rng(seed).uniform(size=(nnodes, dim))
    if k is None:
        k = np.sqrt(1.0 / nnodes)
    fixed = list(fixed)
    t = 0.1
    dt = t / float(iterations + 1)
    disp = np.zeros((dim, nnodes))
    for _ in range(iterations):
        disp *= 0
        for i in range(nnodes):
            if i in fixed:
                continue
            disp[:, i] += displacement(pos, W, k, i)
        length = np.sqrt((disp ** 2).sum(axis=0))
        length = np.where(length < 0.01, 0.1, length)
        pos += (disp * t / length).T
        t -= dt
    return pos


def temperatures(iterations):
    """The temperature of each iteration (_layout.py:190-191, 217)."""
    t, dt, out = 0.1, 0.1 / float(iterations + 1), []
    for _ in range(iterations):
        out.append(t)
        t -= dt
    return out


def rescale(pos, scale=1):
    """_rescale_layout (_layout.py:222-233), in place."""
    lim = 0
    for i in range(pos.shape[1]):
        pos[:, i] -= pos[:, i].mean()
        lim = max(pos[:, i].max(), lim)
    for i in range(pos.shape[1]):
        pos[:, i] *= scale / lim
    return pos


def fruchterman_reingold(W, dim=2, k=None, pos=None, fixed=[], iterations=50, scale=1.0,
                         center=None, seed=None):
    """``G.set_coordinates('spring', seed, **kwargs)`` of a graph with adjacency W
    (_layout.py:121-166)."""
    n = W.shape[0]
    if center is None or np.shape(center)[1] != dim:
        center = np.zeros((1, dim))
    if pos is None:
        dom_size = 1
        start = None
    else:
        dom_size = np.max(pos)
        start = np.random.default_rng(seed).uniform(size=(n, dim)) * dom_size + center
        for i in range(n):
            start[i] = np.asanyarray(pos[i])
    if k is None and len(fixed) > 0:
        k = dom_size / np.sqrt(n)
    out = run(W, dim, k, start, fixed, iterations, seed)
    if len(fixed) == 0:
        out = rescale(out, scale=scale) + center
    return out


def _magnitudes(pos, W, k, rows):
    """S[r, a] = sum_j |delta_ija| (k^2 / d_ij^2 + A_ij d_ij / |k|) for i = rows[r]."""
    n, dim = pos.shape
    out = np.zeros((len(rows), dim))
    block = max(1, (1 << 22) // max(n * dim, 1))
    for s in range(0, len(rows), block):
        r = rows[s:s + block]
        delta = pos[r, None, :] - pos[None, :, :]
        d = np.maximum(np.sqrt((delta ** 2).sum(axis=2)), 0.01)
        A = np.zeros((len(r), n))
        for c, i in enumerate(r):
            A[c] = _adjacency_row(W, i)[0]
        out[s:s + len(r)] = (np.abs(delta) * (k * k / d ** 2 + A * d / abs(k))[:, :, None]).sum(1)
    return out


def step_bound(pos, W, k, t, fixed=(), rows=None):
    r"""One step of ``rows`` with a bound on any reordering of its sums.

    Returns ``(new, alt, bound)``, each (len(rows), dim): ``new`` is :func:`step`; a result
    ``y`` of row i is correct when ``|y - new| <= bound`` in every component, or
    ``|y - alt| <= bound`` in every component (:func:`within`).  ``alt`` is the other branch of
    the length test where the test is decided by rounding, ``new`` elsewhere.

    Derivation.  u = 2^-53.  For vertex i let S_a = sum_j |delta_ija| (k^2/d_ij^2 + A_ij d_ij/|k|)
    (:func:`_magnitudes`).  Each term delta (k^2/d^2 - A d/k) passes through at most 2 dim + 12
    roundings (the difference, the squares and their sum, sqrt, the clamp, the reciprocal or
    division, the products) -- the device's reciprocal is within 3 u of 1/d^2 -- and the sum of at
    most 2 N terms (repulsion and attraction, summed together or apart, in any order) adds at
    most 2 N roundings, so any evaluation of disp_ia is within gamma_m S_a of the exact value,
    m = 2 N + 2 dim + 16, gamma_m = m u / (1 - m u).  Two evaluations are within E_a = 2 gamma_m S_a
    of each other, and their lengths within r = |E| + 2 (dim + 2) u L, L the reference's length.

    * L - r >= 0.01: both divide by the length, and |a/|a| - b/|b|| <= 2 |a - b| / |b|, so the
      moves differ by at most t min(2 |E| / L, 2).
    * L + r < 0.01: both divide by 0.1: the moves differ by at most t E_a / 0.1.
    * otherwise either branch may be taken: both results are accepted, each within the larger
      of the two bounds.

    The update p + (disp t) / length rounds three times on each side, and the length carries
    (dim + 2) u more: 4 u |new| + (2 dim + 12) u t is added.  Fixed vertices have bound 0: they
    must not move.  The bound grows as 1/L where the forces cancel -- where the layout is
    chaotic.
    """
    W = sparse.csr_matrix(W)
    n, dim = pos.shape
    rows = np.arange(n) if rows is None else np.asarray(rows)
    fixed = list(fixed)
    moving = np.array([i not in fixed for i in rows], dtype=bool)
    disp = np.zeros((dim, len(rows)))
    for c, i in enumerate(rows):
        if moving[c]:
            disp[:, c] += displacement(pos, W, k, i)
    new = _move(pos[rows], disp, t)

    m = 2 * n + 2 * dim + 16
    gamma = m * U / (1 - m * U)
    E = 2 * gamma * _magnitudes(pos, W, k, rows)                    # (rows, dim)
    E2 = np.sqrt((E ** 2).sum(axis=1))
    L = np.sqrt((disp ** 2).sum(axis=0))
    r = E2 + 2 * (dim + 2) * U * L
    with np.errstate(divide="ignore", invalid="ignore"):
        b_norm = t * np.minimum(np.where(L > 0, 2 * E2 / L, np.inf), 2.0)
    b_norm = b_norm[:, None] * np.ones((1, dim))
    b_small = t * E / 0.1
    normal_sure = L - r >= 0.01
    small_sure = L + r < 0.01
    either = ~normal_sure & ~small_sure
    bound = np.where(normal_sure[:, None], b_norm, b_small)
    bound = np.where(either[:, None], np.maximum(b_norm, b_small), bound)
    bound += 4 * U * np.abs(new) + (2 * dim + 12) * U * t

    alt = new.copy()
    took_normal = L >= 0.01
    other = np.where(took_normal, 0.1, np.where(L > 0, L, 0.1))
    alt_rows = either & moving
    alt[alt_rows] = pos[rows][alt_rows] + (disp[:, alt_rows] * t / other[alt_rows]).T

    bound[~moving] = 0.0
    return new, alt, bound


def within(got, new, alt, bound):
    """Per row: every component within ``bound`` of ``new``, or every component of ``alt``."""
    return (np.abs(got - new) <= bound).all(axis=1) | (np.abs(got - alt) <= bound).all(axis=1)
