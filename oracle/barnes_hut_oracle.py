r"""NumPy restatement of the Barnes-Hut spring repulsion (csrc/barnes_hut.cu), with a proven
bound on the error of each vertex's sum.

TEST INFRASTRUCTURE ONLY: nothing under ``pygsp_b200/`` imports this module.

:func:`build_tree` restates the device's tree: Morton keys by ``graphs.morton_order``'s formula
(21 bits per axis, float64 quantisation, truncated and clamped), a stable sort, Karras's binary
radix tree over the sorted keys with a duplicate key broken by its sorted index (the same
topology and node numbering), and each internal node's count, axis-aligned bounding box (AABB)
and centroid.  The AABBs are min / max, so they are the device's bits; the centroids are
``c_L + (M_R / M) (c_R - c_L)``, the device's formula, which differ from it by the fma's rounding.

:func:`walk` walks the tree for given query rows with a slightly relaxed acceptance rule and
returns the Barnes-Hut force of its frontier, the frontier bound and visit counts.
:func:`bh_step_bound` is ``layout_oracle.step_bound``'s case analysis with that bound added to the
displacement error.
"""
import numpy as np
from scipy import sparse

from . import layout_oracle as lo

BITS = 21                    # Morton bits per axis (dim <= 3)
STACK = 96                   # the device walk's stack entries
MIN_D2 = 0.01 ** 2
ETA = 1e-10                  # relative margin of the relaxed acceptance and of the bound
TINY = 1e-290                # absolute margin of the acceptance (underflow of D^2)
U = lo.U


def morton_keys(pos):
    """The uint64 Morton code of every row (graphs.morton_order's integer codes; a NaN gives 0)."""
    pos = np.asarray(pos, dtype=np.float64)
    n, d = pos.shape
    lo_ = pos.min(axis=0)
    span = np.maximum(pos.max(axis=0) - lo_, 1e-300)
    with np.errstate(invalid="ignore"):
        v = (pos - lo_) / span * float(1 << BITS)
        v = np.where(v > 0, v, 0.0)
        q = np.minimum(v, float((1 << BITS) - 1)).astype(np.uint64)
    code = np.zeros(n, dtype=np.uint64)
    for b in range(BITS):
        for k in range(d):
            code |= ((q[:, k] >> np.uint64(b)) & np.uint64(1)) << np.uint64(b * d + k)
    return code


def _bitlen32(v):
    """Bit length of non-negative integers below 2^32 (exact: float64 holds them)."""
    return np.frexp(v.astype(np.float64))[1].astype(np.int64)


def _delta(keys, i, j):
    """Common prefix length of the extended keys (keys[i], i) and (keys[j], j); -1 where j is
    outside [0, n) (the device's bh_delta)."""
    n = len(keys)
    out = np.full(i.shape, -1, dtype=np.int64)
    ok = (j >= 0) & (j < n)
    a, b = keys[i[ok]], keys[j[ok]]
    x = a ^ b
    hi = (x >> np.uint64(32)).astype(np.int64)
    lo32 = (x & np.uint64(0xFFFFFFFF)).astype(np.int64)
    bl = np.where(hi > 0, 32 + _bitlen32(hi), _bitlen32(lo32))
    same = 64 + 32 - _bitlen32(i[ok] ^ j[ok])
    out[ok] = np.where(x != 0, 64 - bl, same)
    return out


def build_tree(pos):
    """The device's tree of the (n, dim) positions as a dict of arrays:

    ``ids`` (sorted index -> vertex), ``keys`` (sorted), ``spos`` (positions in sorted order),
    and per internal node v < n - 1: ``left`` / ``right`` (w >= 0 internal node w, w < 0 the leaf
    at sorted index ~w), ``first`` / ``last`` (its range of sorted indices), ``count``, ``lo`` /
    ``hi`` (AABB), ``centroid``, ``depth`` (root 0), ``Q`` (an upper bound on sum |y - c|^2 over
    the node's points y, c their exact centroid, that covers the centroids' rounding);
    ``height`` is the largest number of internal nodes on a root-to-leaf path."""
    pos = np.asarray(pos, dtype=np.float64)
    n, dim = pos.shape
    keys = morton_keys(pos)
    ids = np.argsort(keys, kind="stable")
    skeys, spos = keys[ids], pos[ids]
    t = dict(ids=ids.astype(np.int32), keys=skeys, spos=spos, n=n, dim=dim)
    m = max(n - 1, 0)
    if n <= 1:
        t.update(left=np.zeros(0, np.int64), right=np.zeros(0, np.int64),
                 first=np.zeros(0, np.int64), last=np.zeros(0, np.int64),
                 count=np.zeros(0, np.int64), lo=np.zeros((0, dim)), hi=np.zeros((0, dim)),
                 centroid=np.zeros((0, dim)), depth=np.zeros(0, np.int64),
                 Q=np.zeros(0), height=0)
        return t
    i = np.arange(m, dtype=np.int64)
    d = np.where(_delta(skeys, i, i + 1) - _delta(skeys, i, i - 1) > 0, 1, -1)
    dmin = _delta(skeys, i, i - d)
    lmax = np.full(m, 2, dtype=np.int64)
    grow = _delta(skeys, i, i + lmax * d) > dmin
    while grow.any():
        lmax[grow] *= 2
        grow &= _delta(skeys, i, i + lmax * d) > dmin
    l = np.zeros(m, dtype=np.int64)
    step = lmax // 2
    while (step >= 1).any():
        take = (step >= 1) & (_delta(skeys, i, i + (l + step) * d) > dmin)
        l += np.where(take, step, 0)
        step //= 2
    j = i + l * d
    dnode = _delta(skeys, i, j)
    s = np.zeros(m, dtype=np.int64)
    step = l.copy()
    active = np.ones(m, dtype=bool)
    while active.any():                      # do { t = ceil(t / 2); ... } while (t > 1)
        step = np.where(active, (step + 1) // 2, step)
        take = active & (_delta(skeys, i, i + (s + step) * d) > dnode)
        s += np.where(take, step, 0)
        active &= step > 1
    g = i + s * d + np.minimum(d, 0)
    first, last = np.minimum(i, j), np.maximum(i, j)
    left = np.where(first == g, ~g, g)
    right = np.where(last == g + 1, ~(g + 1), g + 1)

    # depth top-down, then the aggregates bottom-up, one level at a time
    depth = np.full(m, -1, dtype=np.int64)
    level, cur = 0, np.array([0])
    while cur.size:
        depth[cur] = level
        ch = np.concatenate([left[cur], right[cur]])
        cur, level = ch[ch >= 0], level + 1
    count = np.zeros(m, dtype=np.int64)
    blo, bhi, cen = np.zeros((m, dim)), np.zeros((m, dim)), np.zeros((m, dim))
    Q = np.zeros(m)

    def child(w):
        leaf = w < 0
        sidx = np.where(leaf, ~w, 0)
        widx = np.where(leaf, 0, w)
        cnt = np.where(leaf, 1, count[widx])
        p = spos[sidx]
        return (cnt, np.where(leaf[:, None], p, blo[widx]), np.where(leaf[:, None], p, bhi[widx]),
                np.where(leaf[:, None], p, cen[widx]))

    for lev in range(level - 1, -1, -1):
        v = np.flatnonzero(depth == lev)
        mL, loL, hiL, cL = child(left[v])
        mR, loR, hiR, cR = child(right[v])
        mm = mL + mR
        w = (mR.astype(np.float64) / mm.astype(np.float64))[:, None]
        count[v] = mm
        blo[v] = np.minimum(loL, loR)
        bhi[v] = np.maximum(hiL, hiR)
        cen[v] = cL + w * (cR - cL)
        # Q <= Q_L + Q_R + M_L (|c_L - c| + 2 delta)^2 + M_R (|c_R - c| + 2 delta)^2: the
        # parallel-axis identity with every centroid off its exact value by at most delta
        dv = _centroid_error(blo[v], bhi[v], dim)
        qL = np.where(left[v] < 0, 0.0, Q[np.maximum(left[v], 0)])
        qR = np.where(right[v] < 0, 0.0, Q[np.maximum(right[v], 0)])
        aL = np.sqrt(((cL - cen[v]) ** 2).sum(axis=1)) + 2 * dv
        aR = np.sqrt(((cR - cen[v]) ** 2).sum(axis=1)) + 2 * dv
        Q[v] = (qL + qR + mL * aL ** 2 + mR * aR ** 2) * (1 + ETA)
    t.update(left=left, right=right, first=first, last=last, count=count, lo=blo, hi=bhi,
             centroid=cen, depth=depth, Q=Q, height=level)
    return t


def _centroid_error(blo, bhi, dim):
    """Bound on |c~ - c| of nodes with these AABBs (see :func:`bh_step_bound`)."""
    maxabs = np.maximum(np.abs(blo), np.abs(bhi)).max(axis=1)
    diag = np.sqrt(((bhi - blo) ** 2).sum(axis=1))
    return STACK * 4 * U * np.sqrt(dim) * (maxabs + diag) * (1 + ETA)


def _f(r):
    """f(r) = r / max(|r|^2, 0.01^2), row-wise."""
    return r / np.maximum((r * r).sum(axis=1), MIN_D2)[:, None]


def walk(tree, x, theta, relax=True, keep_frontier=False):
    r"""Barnes-Hut walk of ``tree`` for the query points ``x`` (R, dim).

    Acceptance: a node whose AABB is one point, or with rho^2 >= 0.01^2 (1 - eta) and
    D^2 <= theta^2 rho^2 (1 + eta) + 1e-290, where eta = 1e-10 when ``relax`` (0 otherwise).  The
    relaxed rule accepts every node the device accepts (see :func:`bh_step_bound`).

    Returns a dict of per-row arrays: ``force`` (R, dim) = the frontier's sum of M f(x - c) and
    of f(x - y) over its leaves, without k^2; ``bound`` = sum over accepted nodes of Q / rho^3
    (rho >= 0.01) or M D / 0.01^2 (rho just below 0.01); ``centroid`` = the centroid-rounding
    term sum M delta_c / max(rho - delta_c, 0.01)^2; ``magnitude`` (R, dim) = sum of |terms|;
    ``cells`` / ``leaves`` visited.  With ``keep_frontier``, ``frontier`` is a list of
    (row, node) pairs: node >= 0 an accepted internal node, node < 0 a leaf ~node.
    """
    x = np.asarray(x, dtype=np.float64)
    R, dim = x.shape
    n = tree["n"]
    eta = ETA if relax else 0.0
    out = dict(force=np.zeros((R, dim)), bound=np.zeros(R), centroid=np.zeros(R),
               magnitude=np.zeros((R, dim)), cells=np.zeros(R, np.int64),
               leaves=np.zeros(R, np.int64))
    frontier = []
    rows = np.arange(R)
    nodes = np.full(R, 0 if n > 1 else ~0, dtype=np.int64)
    spos = tree["spos"]
    while rows.size:
        leaf = nodes < 0
        lr, ls = rows[leaf], ~nodes[leaf]
        term = _f(x[lr] - spos[ls])
        np.add.at(out["force"], lr, term)
        np.add.at(out["magnitude"], lr, np.abs(term))
        np.add.at(out["leaves"], lr, 1)
        if keep_frontier:
            frontier += list(zip(lr.tolist(), (~ls).tolist()))
        ir, iv = rows[~leaf], nodes[~leaf]
        np.add.at(out["cells"], ir, 1)
        blo, bhi, xx = tree["lo"][iv], tree["hi"][iv], x[ir]
        e = bhi - blo
        diag2 = (e * e).sum(axis=1)
        gap = np.maximum(np.maximum(blo - xx, xx - bhi), 0.0)
        rho2 = (gap * gap).sum(axis=1)
        point = (blo == bhi).all(axis=1)
        acc = point | ((rho2 >= MIN_D2 * (1 - eta))
                       & (diag2 <= theta * theta * rho2 * (1 + eta) + TINY))
        ar, av = ir[acc], iv[acc]
        M = tree["count"][av].astype(np.float64)
        c = tree["centroid"][av]
        term = M[:, None] * _f(x[ar] - c)
        np.add.at(out["force"], ar, term)
        np.add.at(out["magnitude"], ar, np.abs(term))
        if keep_frontier:
            frontier += list(zip(ar.tolist(), av.tolist()))
        # the bound of each accepted node that is not one point
        pt = point[acc]
        rho = np.sqrt(rho2[acc]) * (1 - ETA)
        D = np.sqrt(diag2[acc]) * (1 + ETA)
        Q = tree["Q"][av] * (1 + ETA)
        with np.errstate(divide="ignore", invalid="ignore"):
            taylor = np.where(rho >= 0.01, Q / rho ** 3, M * D / MIN_D2)
        taylor = np.where(pt, 0.0, taylor)
        dc = _centroid_error(tree["lo"][av], tree["hi"][av], dim)
        cterm = np.where(pt, 0.0, M * dc / np.maximum(rho - dc, 0.01) ** 2)
        np.add.at(out["bound"], ar, taylor)
        np.add.at(out["centroid"], ar, cterm)
        orows, ov = ir[~acc], iv[~acc]
        rows = np.concatenate([orows, orows])
        nodes = np.concatenate([tree["left"][ov], tree["right"][ov]])
    if keep_frontier:
        out["frontier"] = frontier
    return out


def exact_repulsion(pos, x):
    """sum_j f(x - p_j) over all points for each query row of x (float64, no k^2)."""
    pos = np.asarray(pos, dtype=np.float64)
    out = np.zeros_like(x)
    for r in range(len(x)):
        out[r] = _f(x[r] - pos).sum(axis=0)
    return out


def bh_step_bound(pos, W, k, t, theta, fixed=(), rows=None, tree=None):
    r"""One step of ``rows`` with a bound that holds for the device's Barnes-Hut step.

    Returns ``(new, alt, bound)`` as ``layout_oracle.step_bound`` does (``new`` is the exact
    reference step; test with ``layout_oracle.within``), for the device's walk of ``tree`` (by
    default the tree of ``pos``) at ``theta``.

    Derivation.  Write f(r) = r / max(|r|^2, 0.01^2) and u = 2^-53.

    * Taylor.  For |r| >= 0.01, f(r) = r / |r|^2 and |D^2 f(r)[h, h]| = 2 |h|^2 / |r|^3 in any
      dimension.  For a cell of points y_j with exact centroid c, AABB at distance rho >= 0.01
      from x, every segment from x - c to x - y_j lies in x - AABB, at distance >= rho from 0, so
      Taylor's theorem about c (the first-order term sum_j Df (y_j - c) vanishes at the
      centroid) gives |sum_j f(x - y_j) - M f(x - c)| <= Q / rho^3, Q = sum_j |y_j - c|^2.
      Opening a cell never increases this: Q_L + Q_R <= Q (parallel-axis identity) and the
      children's rho are >= rho; a cell of one point (D = 0) and a leaf have error 0.
    * The clamp.  When rho is just below 0.01 f is clamped on part of the AABB; f is Lipschitz
      with constant 1 / 0.01^2 everywhere, so a cell's error is at most M D / 0.01^2, and the
      cells below it that the device may accept instead add up to at most the same (their M D
      sum to at most M D).
    * Relaxation.  The device accepts when fl(D^2) <= fl(fl(theta^2) fl(rho^2)) and
      fl(rho^2) >= 0.01^2: D^2 and rho^2 are sums of at most 3 squares of exact-sign
      differences (at most 5 roundings each), so the exact quantities satisfy the test within a
      relative 16 u.  :func:`walk` accepts with a relative margin eta = 1e-10 >> 16 u (and an
      absolute 1e-290 for D^2 that underflows), so every node the device accepts is accepted by
      the oracle or lies below a node the oracle accepts: the oracle's frontier is a cut above
      the device's.  By the two monotonicity facts above, the oracle's sum over its frontier of
      Q / rho^3 (rho >= 0.01, rho taken as sqrt(fl(rho^2)) (1 - eta)) or M D / 0.01^2 (the band
      just below 0.01) bounds the device's approximation error, whichever near-threshold nodes
      it opened.  Q and D are enlarged by (1 + eta) for their own rounding.
    * Centroid rounding.  The device's centroid c~ = fl(fma(M_R / M, c_R - c_L, c_L)) adds at
      most 2 u D + u max|coordinate| per level to its children's error, over at most 94 levels:
      |c~ - c| <= delta = 96 * 4 u sqrt(dim) (max|coordinate| + D).  f is 1 / max(rho - delta,
      0.01)^2-Lipschitz between x - c and x - c~, so each accepted cell adds M delta /
      max(rho - delta, 0.01)^2, a quantity that also only shrinks under opening.  A cell of
      coincident points has c~ = c exactly.
    * Evaluation.  The device's terms are the all-pairs terms regrouped; each monopole's
      magnitude is at most the sum of its points' magnitudes plus its error, so the device's own
      rounding is at most gamma_m (S_a + k^2 (B + C)), gamma_m and S_a those of ``step_bound``
      (the monopole term has one rounding more than a pair term, within m's slack).

    So the device's displacement differs from the reference's by at most
    E_a = 2 gamma_m S_a + k^2 (B + C) (1 + gamma_m), B the frontier bound and C the centroid
    term, and ``step_bound``'s case analysis on the length test and its update rounding apply
    with this E.  Fixed vertices have bound 0.
    """
    W = sparse.csr_matrix(W)
    pos = np.asarray(pos, dtype=np.float64)
    n, dim = pos.shape
    rows = np.arange(n) if rows is None else np.asarray(rows)
    if tree is None:
        tree = build_tree(pos)
    fixed = list(fixed)
    moving = np.array([i not in fixed for i in rows], dtype=bool)
    disp = np.zeros((dim, len(rows)))
    for c, i in enumerate(rows):
        if moving[c]:
            disp[:, c] += lo.displacement(pos, W, k, i)
    new = lo._move(pos[rows], disp, t)

    m = 2 * n + 2 * dim + 16
    gamma = m * U / (1 - m * U)
    wk = walk(tree, pos[rows], theta)
    extra = k * k * (wk["bound"] + wk["centroid"]) * (1 + gamma)
    E = 2 * gamma * lo._magnitudes(pos, W, k, rows) + extra[:, None]
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
