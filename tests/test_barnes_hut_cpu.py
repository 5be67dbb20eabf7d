"""The Barnes-Hut oracle on the CPU (oracle/barnes_hut_oracle.py): its tree has the documented
invariants and the device's Morton order, its frontier force lies within its own bound of the
exact repulsion on random, clustered, collinear and duplicated clouds, and the bound rejects the
usual Barnes-Hut mistakes."""
import numpy as np
import pytest

from oracle import barnes_hut_oracle as bo
from pygsp_b200.graphs.generators import morton_order

U = np.finfo(np.float64).eps / 2


def _cloud(kind, n, dim, seed):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.uniform(size=(n, dim))
    if kind == "clustered":
        centres = rng.uniform(-5, 5, size=(4, dim))
        scale = np.array([1e-3, 1e-1, 1.0, 1e-6])
        lab = rng.integers(0, 4, size=n)
        return centres[lab] + scale[lab, None] * rng.standard_normal((n, dim))
    if kind == "collinear":
        t = rng.uniform(-3, 3, size=n)
        direction = np.arange(1, dim + 1, dtype=np.float64)
        return t[:, None] * direction[None, :] + 0.5
    if kind == "duplicated":
        base = rng.uniform(size=(n // 4, dim))
        return base[rng.integers(0, len(base), size=n)]
    raise ValueError(kind)


def _ranges(t, w):
    return (~w, ~w) if w < 0 else (t["first"][w], t["last"][w])


def _check_invariants(t):
    n = t["n"]
    for v in range(n - 1):
        a, b = _ranges(t, t["left"][v]), _ranges(t, t["right"][v])
        assert a[0] == t["first"][v] and b[1] == t["last"][v] and a[1] + 1 == b[0], v
        assert t["count"][v] == t["last"][v] - t["first"][v] + 1
        pts = t["spos"][t["first"][v]:t["last"][v] + 1]
        np.testing.assert_array_equal(t["lo"][v], pts.min(axis=0))
        np.testing.assert_array_equal(t["hi"][v], pts.max(axis=0))
    if n > 1:
        assert t["first"][0] == 0 and t["last"][0] == n - 1
    # every sorted index is a leaf of exactly one node
    leaves = np.concatenate([~t["left"][t["left"] < 0], ~t["right"][t["right"] < 0]])
    np.testing.assert_array_equal(np.sort(leaves), np.arange(n) if n > 1 else [])
    assert np.all(np.diff(t["keys"].astype(np.float64)) >= 0)


@pytest.mark.parametrize("dim", [1, 2, 3])
@pytest.mark.parametrize("kind", ["random", "clustered", "collinear", "duplicated"])
def test_tree_invariants(kind, dim):
    t = bo.build_tree(_cloud(kind, 400, dim, 7))
    _check_invariants(t)
    assert t["height"] <= 94


@pytest.mark.parametrize("dim", [2, 3])
def test_keys_are_morton_orders(dim):
    p = _cloud("clustered", 3000, dim, 3)
    np.testing.assert_array_equal(bo.build_tree(p)["ids"], morton_order(p))


def test_depth_on_degenerate_clouds():
    t = bo.build_tree(np.zeros((5000, 3)))
    _check_invariants(t)
    assert t["height"] <= 94 and (t["keys"] == 0).all()
    rng = np.random.default_rng(1)
    cloud = rng.uniform(-5e5, 5e5, size=(3000, 2))
    cluster = 1e-12 * rng.standard_normal((2000, 2)) + 123.25
    t = bo.build_tree(np.vstack([cloud, cluster]))
    _check_invariants(t)
    assert t["height"] <= 94
    # a cell of coincident points has their exact centroid
    t = bo.build_tree(np.vstack([np.full((7, 2), 0.3), [[1.0, 2.0]]]))
    point = (t["lo"] == t["hi"]).all(axis=1)
    assert point.any()
    np.testing.assert_array_equal(t["centroid"][point], 0.3)


def test_one_two_and_nan():
    t = bo.build_tree(np.array([[0.5, 0.5]]))
    assert t["height"] == 0 and len(t["left"]) == 0
    w = bo.walk(t, np.array([[0.5, 0.5]]), 0.5)
    assert (w["force"] == 0).all() and w["leaves"][0] == 1
    t = bo.build_tree(np.array([[0.0], [1.0]]))
    assert t["left"][0] == ~0 and t["right"][0] == ~1
    keys = bo.morton_keys(np.array([[np.nan, 0.0], [1.0, 1.0], [0.0, 2.0]]))
    assert keys.dtype == np.uint64 and np.isfinite(keys.astype(np.float64)).all()


@pytest.mark.parametrize("theta", [0.25, 0.5, 1.0])
@pytest.mark.parametrize("dim", [1, 2, 3])
@pytest.mark.parametrize("kind", ["random", "clustered", "collinear", "duplicated"])
def test_force_within_its_frontier_bound(kind, dim, theta):
    p = _cloud(kind, 600, dim, 11)
    t = bo.build_tree(p)
    rows = np.arange(0, 600, 7)
    w = bo.walk(t, p[rows], theta)
    exact = bo.exact_repulsion(p, p[rows])
    err = np.sqrt(((w["force"] - exact) ** 2).sum(axis=1))
    # both sums round: the frontier's at most len(p) terms, the exact one's len(p) terms
    slack = 4 * len(p) * U * np.sqrt((w["magnitude"] ** 2).sum(axis=1) * dim)
    assert (err <= w["bound"] + w["centroid"] + slack).all(), (err - w["bound"]).max()
    assert (w["leaves"] + w["cells"] <= 2 * len(p)).all()


def test_theta_zero_opens_every_cell_of_distinct_points():
    p = _cloud("random", 300, 2, 2)
    w = bo.walk(bo.build_tree(p), p[:20], 0.0, relax=False)
    assert (w["leaves"] == 300).all() and (w["bound"] == 0).all()


# ----------------------------------------------------------------- the bound is not vacuous
def _setup():
    rng = np.random.default_rng(5)
    a = 10.0 + 0.05 * rng.uniform(size=(9, 2))
    b = np.array([[-10.0, 0.0]]) + 0.05 * rng.uniform(size=(10, 2))
    p = np.vstack([[[0.0, 0.0]], a, [[11.0, 1.0]], b])
    t = bo.build_tree(p)
    w = bo.walk(t, p[:1], 0.5, keep_frontier=True)
    exact = bo.exact_repulsion(p, p[:1])[0]
    cells = [v for r, v in w["frontier"] if v >= 0 and not (t["lo"][v] == t["hi"][v]).all()]
    assert cells, "the configuration must accept a cell of distinct points"
    assert np.linalg.norm(w["force"][0] - exact) <= w["bound"][0] + w["centroid"][0] + 1e-12
    return p, t, w, exact, cells


def _mono(t, v, x, c=None):
    c = t["centroid"][v] if c is None else c
    return t["count"][v] * bo._f((x - c)[None, :])[0]


def _rejected(got, exact, w):
    return np.linalg.norm(got - exact) > w["bound"][0] + w["centroid"][0]


def test_bound_rejects_a_dropped_cell():
    p, t, w, exact, cells = _setup()
    assert _rejected(w["force"][0] - _mono(t, cells[0], p[0]), exact, w)


def test_bound_rejects_a_cell_counted_twice():
    p, t, w, exact, cells = _setup()
    assert _rejected(w["force"][0] + _mono(t, cells[0], p[0]), exact, w)


def test_bound_rejects_the_monopole_at_the_box_centre():
    p, t, w, exact, cells = _setup()
    got = w["force"][0].copy()
    for v in cells:
        centre = 0.5 * (t["lo"][v] + t["hi"][v])
        got += _mono(t, v, p[0], centre) - _mono(t, v, p[0])
    assert _rejected(got, exact, w)


def test_bound_rejects_a_cell_accepted_around_the_query():
    p, t, w, exact, cells = _setup()
    assert (t["lo"][0] <= p[0]).all() and (p[0] <= t["hi"][0]).all()
    assert _rejected(_mono(t, 0, p[0]), exact, w)


def test_bh_step_bound_contains_the_exact_step():
    from oracle import layout_oracle as lo
    from scipy import sparse
    p = _cloud("clustered", 200, 2, 9)
    W = sparse.random(200, 200, density=0.03, random_state=1)
    W = sparse.csr_matrix(W + W.T)
    k = np.sqrt(1 / 200)
    new0, _, b0 = lo.step_bound(p, W, k, 0.1)
    new, alt, b = bo.bh_step_bound(p, W, k, 0.1, 0.5)
    np.testing.assert_array_equal(new, new0)
    assert (b >= b0).all()
    assert lo.within(new, new, alt, b).all()


def test_bh_step_bound_is_step_bound_without_an_approximation():
    """At theta = 0 on distinct points the frontier is every leaf and adds nothing, so the case
    analysis bh_step_bound restates must give step_bound's results bit for bit."""
    from oracle import layout_oracle as lo
    from scipy import sparse
    for seed, fixed in ((3, ()), (4, (0, 7, 50))):
        p = _cloud("random", 150, 2, seed)
        W = sparse.random(150, 150, density=0.05, random_state=seed)
        W = sparse.csr_matrix(W + W.T)
        k = np.sqrt(1 / 150)
        for t in (0.1, 1e-4):
            want = lo.step_bound(p, W, k, t, fixed=fixed)
            got = bo.bh_step_bound(p, W, k, t, 0.0, fixed=fixed)
            for a, b in zip(got, want):
                np.testing.assert_array_equal(a, b)
