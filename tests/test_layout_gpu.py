"""Vertex coordinates on the device (graphs/layout.py, csrc/layout.cu): every spring step against
the float64 restatement of the reference's step and its bound (oracle/layout_oracle.py), short
runs and set_coordinates against tests/golden/layout.npz (the unmodified PyGSP 0.6.1), run-to-run
determinism, fixed vertices, the generic dimension, awkward sizes and the host kinds."""
import json

import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from, load_golden
from oracle import layout_oracle as lo

pytestmark = pytest.mark.gpu

GOLD = load_golden("layout")
GRAPHS = [str(g) for g in GOLD["graphs"]]
SC_CASES = [str(c) for c in GOLD["sc_names"]]


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


def _graph(gsp, name, dtype=np.float64):
    return gsp.graphs.Graph(_W(name), dtype=dtype)


def _k(n):
    return np.sqrt(1.0 / n)


def _assert_step(got, pos, W, k, t, fixed=(), rows=None, what=""):
    new, alt, bound = lo.step_bound(pos, W, k, t, fixed=fixed, rows=rows)
    ok = lo.within(got, new, alt, bound)
    if not ok.all():
        r = int(np.flatnonzero(~ok)[0])
        raise AssertionError("%s: %d rows outside the bound; first: row %d got %r want %r bound %r"
                             % (what, int((~ok).sum()), r, got[r], new[r], bound[r]))
    return new, alt, bound


def _span(x):
    return float((x.max(axis=0) - x.min(axis=0)).max())


# --------------------------------------------------------------------------- one step
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", GRAPHS)
def test_one_step_from_every_golden_state(gsp, layout, name, dtype):
    G = _graph(gsp, name, dtype)
    W, k = _W(name), _k(G.N)
    for state in ("start", "run10", "run50"):
        pos = GOLD["g_%s_%s" % (name, state)]
        got = layout._spring_step(G, pos, k, 0.1)
        new, alt, bound = _assert_step(got, pos, W, k, 0.1, what=state)
        # the reference's own step lies within the same bound
        assert lo.within(GOLD["g_%s_step_%s" % (name, state)], new, alt, bound).all()
        assert np.isfinite(got).all()


# ---------------------------------------------------------------- every step of a layout
@pytest.mark.parametrize("name", GRAPHS)
def test_every_step_of_a_50_iteration_layout(gsp, layout, name):
    G = _graph(gsp, name)
    W, k = _W(name), _k(G.N)
    start = GOLD["g_%s_start" % name]
    final, states = layout._spring_layout(G, start, k, 50, (), keep_states=True)
    np.testing.assert_array_equal(final, states[-1])
    prev = start
    for it, t in enumerate(lo.temperatures(50)):
        _assert_step(states[it], prev, W, k, t, what="iteration %d" % it)
        prev = states[it]


def test_first_and_last_step_on_a_large_morton_sensor(gsp, layout):
    G = gsp.graphs.Sensor(100000, seed=0, order="morton", dtype=np.float32)
    W = G.W.to_scipy()
    k = _k(G.N)
    start = np.random.default_rng(1).uniform(size=(G.N, 2))
    final, states = layout._spring_layout(G, start, k, 50, (), keep_states=True)
    rows = np.sort(np.random.default_rng(2).choice(G.N, 256, replace=False))
    temps = lo.temperatures(50)
    _assert_step(states[0][rows], start, W, k, temps[0], rows=rows, what="first")
    _assert_step(states[-1][rows], states[-2], W, k, temps[-1], rows=rows, what="last")
    assert np.isfinite(final).all()


# ------------------------------------------------------------------ against the reference
@pytest.mark.parametrize("name", GRAPHS)
def test_short_runs_match_the_reference(gsp, layout, name):
    G = _graph(gsp, name)
    start = GOLD["g_%s_start" % name]
    for it in (1, 2, 10):
        want = GOLD["g_%s_run%d" % (name, it)]
        got = layout._spring_layout(G, start, _k(G.N), it, ())
        tol = 1e-11 * max(_span(want), 1e-300)
        np.testing.assert_allclose(got, want, rtol=0, atol=tol, err_msg="iterations=%d" % it)


@pytest.mark.parametrize("case", SC_CASES)
def test_set_coordinates_matches_the_reference(gsp, case):
    call = json.loads(str(GOLD["sc_%s_call" % case]))
    want = GOLD["sc_" + case]
    G = _graph(gsp, call["graph"])
    kw = dict(call["kwargs"])
    if kw.get("pos") == "pos":
        kw["pos"] = GOLD["sc_%s_pos" % case]
    if call["kind"] == "community2D":
        G.info = {"node_com": GOLD["sbm_node_com"], "comm_sizes": GOLD["sbm_comm_sizes"],
                  "world_rad": GOLD["sbm_world_rad"]}
    G.set_coordinates(call["kind"], seed=call["seed"], **kw)
    got = np.asarray(G.coords)
    assert got.shape == want.shape
    if call["kind"] == "spring" and kw.get("iterations", 50) == 50:
        # 50 iterations of a chaotic map: only the rescale can be compared
        assert np.isfinite(got).all()
        np.testing.assert_allclose(got.mean(axis=0), 0, atol=1e-12)
        assert got.max() == pytest.approx(1.0, abs=1e-12)
    elif call["kind"] == "spring":
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-11 * _span(want))
    elif call["kind"].startswith("laplacian_eigenmap"):
        sign = np.sign((got * want).sum(axis=0))
        np.testing.assert_allclose(got * sign, want, rtol=0, atol=1e-8)
        n = 3 if call["kind"].endswith("2D") else 4
        np.testing.assert_array_equal(got, G.U[:, 1:n])
    else:
        assert got.dtype == want.dtype, (got.dtype, want.dtype)
        np.testing.assert_array_equal(got, want)


# ---------------------------------------------------------------------------- properties
def test_two_runs_are_bit_identical(gsp, layout):
    for name in ("sensor300", "sbm"):
        G = _graph(gsp, name)
        start = GOLD["g_%s_start" % name]
        a = layout._spring_layout(G, start, _k(G.N), 50, ())
        b = layout._spring_layout(G, start, _k(G.N), 50, ())
        np.testing.assert_array_equal(a, b)
    G = gsp.graphs.Sensor(20000, seed=3, order="morton")
    start = np.random.default_rng(3).uniform(size=(G.N, 2))
    a = layout._spring_layout(G, start, _k(G.N), 3, ())
    b = layout._spring_layout(G, start, _k(G.N), 3, ())
    np.testing.assert_array_equal(a, b)


def test_fixed_vertices_and_the_final_rescale(gsp, layout):
    G = _graph(gsp, "sensor300")
    W = _W("sensor300")
    fixed = [0, 5, 17, 299]
    pos = GOLD["sc_spring_fixed_pos"]
    k = np.max(pos) / np.sqrt(G.N)
    final, states = layout._spring_layout(G, pos, k, 10, fixed, keep_states=True)
    np.testing.assert_array_equal(final[fixed], pos[fixed])
    _assert_step(states[0], pos, W, k, 0.1, fixed=fixed, what="fixed")
    G.set_coordinates("spring", seed=4, pos=pos, fixed=fixed, iterations=10)
    np.testing.assert_array_equal(G.coords, final)          # no rescale with fixed vertices

    start = np.random.default_rng(8).uniform(size=(G.N, 2))
    raw = layout._spring_layout(G, start, _k(G.N), 10, ())
    G.set_coordinates("spring", seed=8, iterations=10, scale=2.5, center=[[1.0, -2.0]])
    np.testing.assert_array_equal(G.coords, lo.rescale(raw.copy(), 2.5) + [[1.0, -2.0]])


@pytest.mark.parametrize("dim", [1, 3, 4])
def test_other_dimensions_step_by_step(gsp, layout, dim):
    name = "sensor300"
    G = _graph(gsp, name)
    W, k = _W(name), _k(G.N)
    start = np.random.default_rng(dim).uniform(size=(G.N, dim))
    final, states = layout._spring_layout(G, start, k, 10, (), keep_states=True)
    prev = start
    for it, t in enumerate(lo.temperatures(10)):
        _assert_step(states[it], prev, W, k, t, what="dim %d iteration %d" % (dim, it))
        prev = states[it]
    want = lo.run(W, dim, None, start.copy(), [], 10, None)
    np.testing.assert_allclose(final, want, rtol=0, atol=1e-11 * _span(want))


@pytest.mark.parametrize("n", [1, 2, 255, 257, 4099])
def test_sizes_off_the_tile_and_chunk_grid(gsp, layout, n):
    rng = np.random.default_rng(n)
    if n > 1:
        W = sparse.random(n, n, density=min(1.0, 6.0 / n), random_state=rng)
        W = sparse.triu(W, 1)
        W = sparse.csr_matrix(W + W.T)
    else:
        W = sparse.csr_matrix((1, 1))
    G = gsp.graphs.Graph(W, dtype=np.float64)
    start = rng.uniform(size=(n, 2))
    start[n // 2] = start[0]                                  # a duplicate point
    k = _k(n)
    for t in (0.1, 0.003):
        got = layout._spring_step(G, start, k, t)
        assert np.isfinite(got).all()
        _assert_step(got, start, W, k, t, what="n=%d" % n)


def test_single_vertex_gives_the_reference_nans(gsp):
    G = _graph(gsp, "n1")
    with np.errstate(divide="ignore", invalid="ignore"):
        G.set_coordinates("spring", seed=1)
        want = lo.fruchterman_reingold(_W("n1"), seed=1)
    assert np.isnan(G.coords).all() and np.isnan(want).all()
    assert G.coords.shape == want.shape == (1, 2)


def test_directed_negative_self_loops_and_isolated(gsp, layout):
    # one row by hand: the attraction follows row i of W and only its positive entries
    W = sparse.csr_matrix(np.array([[0.5, 1.0, -2.0, 0.0],
                                    [0.0, 0.0, 0.0, 0.0],
                                    [1.0, 0.0, 0.0, 0.0],
                                    [0.0, 0.0, 0.0, 0.0]]))
    G = gsp.graphs.Graph(W, dtype=np.float64)
    pos = np.array([[0.0, 0.0], [0.3, 0.1], [-0.2, 0.4], [0.5, -0.5]])
    got = layout._spring_step(G, pos, 0.5, 0.1)
    _assert_step(got, pos, W, 0.5, 0.1, what="hand")
    disp = sum((pos[0] - pos[j]) * 0.25 / max(np.linalg.norm(pos[0] - pos[j]), 0.01) ** 2
               for j in range(4))
    disp = disp - (pos[0] - pos[1]) * np.linalg.norm(pos[0] - pos[1]) / 0.5
    np.testing.assert_allclose(got[0], pos[0] + disp * 0.1 / np.linalg.norm(disp), rtol=1e-13,
                               atol=1e-15)


# ----------------------------------------------------------------------------- host kinds
def test_community2d_on_the_package_sbm(gsp):
    G = gsp.graphs.StochasticBlockModel(N=400, k=5, p=0.1, q=0.01, seed=2)
    G.set_coordinates("community2D", seed=5)
    info = G.info
    Nc = info["comm_sizes"].shape[0]
    com = info["world_rad"] * np.array(list(zip(np.cos(2 * np.pi * np.arange(1, Nc + 1) / Nc),
                                                np.sin(2 * np.pi * np.arange(1, Nc + 1) / Nc))))
    coords = np.random.default_rng(5).uniform(size=(G.N, 2))
    coords = np.array([[e[0] * np.cos(2 * np.pi * e[1]), e[0] * np.sin(2 * np.pi * e[1])]
                       for e in coords])
    for i in range(G.N):
        c = info["node_com"][i]
        coords[i] = com[c] + np.sqrt(info["comm_sizes"][c]) * coords[i]
    np.testing.assert_array_equal(G.coords, coords)
    np.testing.assert_array_equal(info["com_coords"], com)

    del G.info["comm_sizes"]
    G.set_coordinates("community2D", seed=5)
    np.testing.assert_array_equal(G.coords, coords)


def test_errors(gsp):
    G = _graph(gsp, "n257")
    with pytest.raises(AttributeError):
        G.set_coordinates("community2D")
    with pytest.raises(ValueError):
        G.set_coordinates("invalid")
    with pytest.raises(ValueError):
        G.set_coordinates(np.zeros((G.N, 4)))
    with pytest.raises(ValueError):
        G.set_coordinates(np.zeros((G.N + 1, 2)))
    G.set_coordinates(np.ones((1, G.N, 3)))
    assert G.coords.shape == (G.N, 3)
    G.set_coordinates(np.arange(G.N))
    assert G.coords.shape == (G.N,)
