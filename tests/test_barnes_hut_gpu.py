"""The Barnes-Hut spring repulsion on the device (csrc/barnes_hut.cu, graphs/layout.py): the tree
against its NumPy restatement, every step against the exact step and the proven bound of
oracle/barnes_hut_oracle.py, theta = 0 against the exact contract, bit-identity, fixed vertices,
the rescale, other dimensions, awkward sizes, degenerate starts and the errors.

Every degenerate cloud goes through the NumPy tree (and its depth check) on the CPU before the
device builds its tree."""
import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from, load_golden
from oracle import barnes_hut_oracle as bo
from oracle import layout_oracle as lo

pytestmark = pytest.mark.gpu

GOLD = load_golden("layout")
GRAPHS = [str(g) for g in GOLD["graphs"]]
BH = dict(repulsion="barnes_hut")


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


@pytest.fixture(scope="module")
def layout(gsp):
    from pygsp_b200.graphs import layout
    return layout


def _W(name):
    return csr_from(GOLD, "g_%s_W" % name)


def _k(n):
    return np.sqrt(1.0 / n)


def _cpu_tree(pos):
    """The NumPy tree of ``pos``, checked before any device call on the same cloud."""
    t = bo.build_tree(pos)
    assert t["height"] <= 94
    n = len(pos)
    if n > 1:
        assert t["first"][0] == 0 and t["last"][0] == n - 1
        assert (t["count"] == t["last"] - t["first"] + 1).all()
    return t


def _device_tree(gsp, pos):
    import torch
    from pygsp_b200 import _native as nat
    n, dim = pos.shape
    m = max(n - 1, 1)
    dev = torch.device("cuda")
    p = torch.as_tensor(np.ascontiguousarray(pos, dtype=np.float64), device=dev)
    ids = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    children = torch.empty(2 * m, dtype=torch.int32, device=dev)
    counts = torch.empty(m, dtype=torch.int32, device=dev)
    boxes = torch.empty(m * 2 * dim, dtype=torch.float64, device=dev)
    cents = torch.empty(m * dim, dtype=torch.float64, device=dev)
    nat.call("gsp_spring_bh_tree", nat.i64(n), nat.i32(dim), p, ids, children, counts, boxes,
             cents, nat.stream_ptr())
    torch.cuda.synchronize()
    n1 = n - 1
    return dict(ids=ids.cpu().numpy()[:n], children=children.cpu().numpy()[:2 * n1],
                counts=counts.cpu().numpy()[:n1], boxes=boxes.cpu().numpy()[:n1 * 2 * dim],
                centroids=cents.cpu().numpy()[:n1 * dim])


def _assert_same_tree(gsp, pos):
    t = _cpu_tree(pos)
    d = _device_tree(gsp, pos)
    n, dim = pos.shape
    np.testing.assert_array_equal(d["ids"], t["ids"])
    if n <= 1:
        return t
    ch = np.stack([t["left"], t["right"]], axis=1).reshape(-1)
    np.testing.assert_array_equal(d["children"], ch)
    np.testing.assert_array_equal(d["counts"], t["count"])
    boxes = d["boxes"].reshape(n - 1, 2, dim)
    np.testing.assert_array_equal(boxes[:, 0], t["lo"])
    np.testing.assert_array_equal(boxes[:, 1], t["hi"])
    tol = 2 * bo._centroid_error(t["lo"], t["hi"], dim)[:, None]
    assert (np.abs(d["centroids"].reshape(n - 1, dim) - t["centroid"]) <= tol).all()
    point = (t["lo"] == t["hi"]).all(axis=1)
    np.testing.assert_array_equal(d["centroids"].reshape(n - 1, dim)[point], t["centroid"][point])
    return t


def _assert_bh_step(got, pos, W, k, t, theta, fixed=(), rows=None, what=""):
    new, alt, bound = bo.bh_step_bound(pos, W, k, t, theta, fixed=fixed, rows=rows)
    ok = lo.within(got, new, alt, bound)
    if not ok.all():
        r = int(np.flatnonzero(~ok)[0])
        raise AssertionError("%s: %d rows outside the bound; first: row %d got %r want %r bound %r"
                             % (what, int((~ok).sum()), r, got[r], new[r], bound[r]))


def _assert_exact_step(got, pos, W, k, t, what=""):
    new, alt, bound = lo.step_bound(pos, W, k, t)
    ok = lo.within(got, new, alt, bound)
    assert ok.all(), "%s: %d rows outside step_bound" % (what, int((~ok).sum()))


def _degenerate(name):
    rng = np.random.default_rng(4)
    if name == "equal":
        return np.full((300, 2), 0.37)
    if name == "collinear":
        t = rng.uniform(size=300)
        return np.stack([t, 2 * t - 0.5], axis=1)
    if name == "cluster_outliers":
        c = 0.5 + 1e-9 * rng.standard_normal((280, 2))
        far = rng.uniform(-1e4, 1e4, size=(20, 2))
        return np.vstack([c, far])
    if name == "tiny_cluster_huge_cloud":
        c = 123.25 + 1e-12 * rng.standard_normal((200, 3))
        return np.vstack([c, rng.uniform(-5e5, 5e5, size=(100, 3))])
    raise ValueError(name)


DEGENERATE = ["equal", "collinear", "cluster_outliers", "tiny_cluster_huge_cloud"]


# ---------------------------------------------------------------------------- the tree
@pytest.mark.parametrize("name", GRAPHS)
def test_tree_matches_numpy_on_golden_states(gsp, name):
    for state in ("start", "run10", "run50"):
        _assert_same_tree(gsp, GOLD["g_%s_%s" % (name, state)])


@pytest.mark.parametrize("name", DEGENERATE)
def test_tree_matches_numpy_on_degenerate_clouds(gsp, name):
    _assert_same_tree(gsp, _degenerate(name))


@pytest.mark.parametrize("dim", [1, 2, 3])
@pytest.mark.parametrize("n", [1, 2, 3, 255, 257, 1000])
def test_tree_matches_numpy_at_small_sizes(gsp, n, dim):
    pos = np.random.default_rng(n + dim).uniform(size=(n, dim))
    if n > 2:
        pos[n // 2] = pos[0]
    _assert_same_tree(gsp, pos)


# ------------------------------------------------------------------- theta = 0: exact contract
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", GRAPHS)
def test_theta_zero_is_within_the_exact_step_bound(gsp, layout, name, dtype):
    G = gsp.graphs.Graph(_W(name), dtype=dtype)
    W, k = _W(name), _k(G.N)
    for state in ("start", "run10", "run50"):
        pos = GOLD["g_%s_%s" % (name, state)]
        got = layout._spring_step(G, pos, k, 0.1, repulsion="barnes_hut", theta=0.0)
        _assert_exact_step(got, pos, W, k, 0.1, what="%s theta=0" % state)


# ---------------------------------------------------------- every step of a BH layout
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("theta", [0.25, 0.5, 1.0])
@pytest.mark.parametrize("name", GRAPHS)
def test_every_step_of_a_50_iteration_bh_layout(gsp, layout, name, theta, dtype):
    G = gsp.graphs.Graph(_W(name), dtype=dtype)
    W, k = _W(name), _k(G.N)
    start = GOLD["g_%s_start" % name]
    final, states = layout._spring_layout(G, start, k, 50, (), keep_states=True, repulsion="barnes_hut",
                                          theta=theta)
    np.testing.assert_array_equal(final, states[-1])
    prev = start
    for it, t in enumerate(lo.temperatures(50)):
        _assert_bh_step(states[it], prev, W, k, t, theta, what="iteration %d" % it)
        prev = states[it]


def test_first_and_last_step_on_a_large_morton_sensor(gsp, layout):
    G = gsp.graphs.Sensor(100000, seed=0, order="morton", dtype=np.float32)
    W = G.W.to_scipy()
    k = _k(G.N)
    start = np.random.default_rng(1).uniform(size=(G.N, 2))
    final, states = layout._spring_layout(G, start, k, 50, (), keep_states=True, **BH)
    rows = np.sort(np.random.default_rng(2).choice(G.N, 256, replace=False))
    temps = lo.temperatures(50)
    _assert_bh_step(states[0][rows], start, W, k, temps[0], 0.5, rows=rows, what="first")
    _assert_bh_step(states[-1][rows], states[-2], W, k, temps[-1], 0.5, rows=rows, what="last")
    assert np.isfinite(final).all()


def test_one_step_on_a_million_vertex_sensor(gsp, layout):
    G = gsp.graphs.Sensor(1000000, seed=0)
    W = G.W.to_scipy()
    k = _k(G.N)
    start = np.random.default_rng(3).uniform(size=(G.N, 2))
    got = layout._spring_step(G, start, k, 0.1, **BH)
    rows = np.sort(np.random.default_rng(4).choice(G.N, 64, replace=False))
    _assert_bh_step(got[rows], start, W, k, 0.1, 0.5, rows=rows, what="1e6")


# ------------------------------------------------------------------------- properties
def test_two_runs_are_bit_identical(gsp, layout):
    G = gsp.graphs.Graph(_W("sbm"))
    start = GOLD["g_sbm_start"]
    a = layout._spring_layout(G, start, _k(G.N), 50, (), **BH)
    b = layout._spring_layout(G, start, _k(G.N), 50, (), **BH)
    np.testing.assert_array_equal(a, b)
    G = gsp.graphs.Sensor(20000, seed=3)
    start = np.random.default_rng(3).uniform(size=(G.N, 2))
    a = layout._spring_layout(G, start, _k(G.N), 3, (), repulsion="barnes_hut", theta=0.7)
    b = layout._spring_layout(G, start, _k(G.N), 3, (), repulsion="barnes_hut", theta=0.7)
    np.testing.assert_array_equal(a, b)


def test_exact_keyword_is_the_default(gsp, layout):
    G = gsp.graphs.Graph(_W("sensor300"))
    start = GOLD["g_sensor300_start"]
    np.testing.assert_array_equal(layout._spring_layout(G, start, _k(G.N), 10, ()),
                                  layout._spring_layout(G, start, _k(G.N), 10, (),
                                                        repulsion="exact"))
    np.testing.assert_array_equal(layout._spring_step(G, start, _k(G.N), 0.1),
                                  layout._spring_step(G, start, _k(G.N), 0.1, repulsion="exact"))
    G.set_coordinates("spring", seed=2)
    a = G.coords
    G.set_coordinates("spring", seed=2, repulsion="exact")
    np.testing.assert_array_equal(a, G.coords)


def test_fixed_vertices_and_the_final_rescale(gsp, layout):
    G = gsp.graphs.Graph(_W("sensor300"))
    W = _W("sensor300")
    fixed = [0, 5, 17, 299]
    pos = GOLD["sc_spring_fixed_pos"]
    k = np.max(pos) / np.sqrt(G.N)
    final, states = layout._spring_layout(G, pos, k, 10, fixed, keep_states=True, **BH)
    np.testing.assert_array_equal(final[fixed], pos[fixed])
    _assert_bh_step(states[0], pos, W, k, 0.1, 0.5, fixed=fixed, what="fixed")
    # the fixed vertices still repel: moving one changes the others' step
    moved = pos.copy()
    moved[5] += 0.3
    other = layout._spring_step(G, moved, k, 0.1, fixed, **BH)
    assert not np.array_equal(other[1], states[0][1])
    G.set_coordinates("spring", seed=4, pos=pos, fixed=fixed, iterations=10, **BH)
    np.testing.assert_array_equal(G.coords, final)

    start = np.random.default_rng(8).uniform(size=(G.N, 2))
    raw = layout._spring_layout(G, start, _k(G.N), 10, (), repulsion="barnes_hut", theta=0.8)
    G.set_coordinates("spring", seed=8, iterations=10, scale=2.5, center=[[1.0, -2.0]],
                      repulsion="barnes_hut", theta=0.8)
    np.testing.assert_array_equal(G.coords, lo.rescale(raw.copy(), 2.5) + [[1.0, -2.0]])


@pytest.mark.parametrize("dim", [1, 3])
def test_other_dimensions_step_by_step(gsp, layout, dim):
    G = gsp.graphs.Graph(_W("sensor300"))
    W, k = _W("sensor300"), _k(G.N)
    start = np.random.default_rng(dim).uniform(size=(G.N, dim))
    final, states = layout._spring_layout(G, start, k, 10, (), keep_states=True, **BH)
    prev = start
    for it, t in enumerate(lo.temperatures(10)):
        _assert_bh_step(states[it], prev, W, k, t, 0.5, what="dim %d iteration %d" % (dim, it))
        prev = states[it]


@pytest.mark.parametrize("n", [1, 2, 3, 127, 129, 255, 257, 4099])
def test_sizes_off_every_block_size(gsp, layout, n):
    rng = np.random.default_rng(n)
    if n > 1:
        W = sparse.random(n, n, density=min(1.0, 6.0 / n), random_state=rng)
        W = sparse.triu(W, 1)
        W = sparse.csr_matrix(W + W.T)
    else:
        W = sparse.csr_matrix((1, 1))
    G = gsp.graphs.Graph(W, dtype=np.float64)
    start = rng.uniform(size=(n, 2))
    start[n // 2] = start[0]
    _cpu_tree(start)
    k = _k(n)
    for t, theta in ((0.1, 0.5), (0.003, 1.0)):
        got = layout._spring_step(G, start, k, t, repulsion="barnes_hut", theta=theta)
        assert np.isfinite(got).all()
        _assert_bh_step(got, start, W, k, t, theta, what="n=%d" % n)


@pytest.mark.parametrize("name", DEGENERATE)
def test_degenerate_starts(gsp, layout, name):
    pos = _degenerate(name)
    _cpu_tree(pos)
    n = len(pos)
    W = sparse.csr_matrix(sparse.diags([np.ones(n - 1), np.ones(n - 1)], [-1, 1]))
    G = gsp.graphs.Graph(W, dtype=np.float64)
    k = _k(n)
    got = layout._spring_step(G, pos, k, 0.1, **BH)
    assert np.isfinite(got).all()
    _assert_bh_step(got, pos, W, k, 0.1, 0.5, what=name)


def test_single_vertex_gives_the_reference_nans(gsp):
    G = gsp.graphs.Graph(_W("n1"))
    with np.errstate(divide="ignore", invalid="ignore"):
        G.set_coordinates("spring", seed=1, **BH)
    assert np.isnan(G.coords).all() and G.coords.shape == (1, 2)


def test_errors(gsp, layout):
    G = gsp.graphs.Graph(_W("n257"))
    with pytest.raises(ValueError):
        G.set_coordinates("spring", theta=0.5)
    with pytest.raises(ValueError):
        G.set_coordinates("spring", repulsion="exact", theta=0.5)
    for theta in (-0.1, np.inf, np.nan):
        with pytest.raises(ValueError):
            G.set_coordinates("spring", repulsion="barnes_hut", theta=theta)
    with pytest.raises(ValueError):
        G.set_coordinates("spring", repulsion="fmm")
    with pytest.raises(ValueError):
        G.set_coordinates("spring", repulsion="barnes_hut", dim=4)
    bad = np.random.default_rng(0).uniform(size=(G.N, 2))
    bad[3, 1] = np.nan
    with pytest.raises(ValueError):
        G.set_coordinates("spring", repulsion="barnes_hut", pos=bad)
    with pytest.raises(ValueError):
        layout._spring_step(G, bad, 0.1, 0.1, repulsion="barnes_hut")
    with pytest.raises(ValueError):
        layout._spring_layout(G, np.zeros((G.N, 4)), 0.1, 2, (), repulsion="barnes_hut")
    with pytest.raises(ValueError):
        layout._spring_step(G, np.zeros((G.N, 2)), 0.1, 0.1, theta=1.0)
