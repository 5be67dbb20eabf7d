"""The float64 restatement of the spring layout (oracle/layout_oracle.py) against
tests/golden/layout.npz (the unmodified PyGSP 0.6.1), and the power of its one-step bound, without
a GPU."""
import json

import numpy as np
import pytest
from scipy import sparse

from conftest import csr_from, load_golden
from oracle import layout_oracle as lo

RUNS = (1, 2, 10, 50)
GOLD = load_golden("layout")
GRAPHS = [str(g) for g in GOLD["graphs"]]
SPRING_CASES = [str(c) for c in GOLD["sc_names"] if str(c).startswith("spring")]


def _graph(name):
    return csr_from(GOLD, "g_%s_W" % name)


@pytest.mark.parametrize("name", GRAPHS)
def test_runs_and_steps_reproduce_golden(name):
    W = _graph(name)
    start = GOLD["g_%s_start" % name]
    for it in RUNS:
        got = lo.run(W, 2, None, start.copy(), [], it, None)
        np.testing.assert_array_equal(got, GOLD["g_%s_run%d" % (name, it)], err_msg=str(it))
    k = np.sqrt(1.0 / W.shape[0])
    for state in ("start", "run10", "run50"):
        got = lo.step(GOLD["g_%s_%s" % (name, state)], W, k, 0.1)
        np.testing.assert_array_equal(got, GOLD["g_%s_step_%s" % (name, state)], err_msg=state)


@pytest.mark.parametrize("case", SPRING_CASES)
def test_set_coordinates_spring_reproduces_golden(case):
    call = json.loads(str(GOLD["sc_%s_call" % case]))
    kw = dict(call["kwargs"])
    if kw.get("pos") == "pos":
        kw["pos"] = GOLD["sc_%s_pos" % case]
    with np.errstate(divide="ignore", invalid="ignore"):
        got = lo.fruchterman_reingold(_graph(call["graph"]), seed=call["seed"], **kw)
    np.testing.assert_array_equal(got, GOLD["sc_" + case])


def test_temperatures_match_the_reference_loop():
    t, dt = 0.1, 0.1 / 51.0
    for i, ti in enumerate(lo.temperatures(50)):
        assert ti == t, i
        t -= dt


@pytest.mark.parametrize("name", ["sensor300", "directed", "dup", "n257"])
@pytest.mark.parametrize("state", ["start", "run10", "run50"])
def test_bound_holds_for_the_reference_step(name, state):
    W = _graph(name)
    k = np.sqrt(1.0 / W.shape[0])
    new, alt, bound = lo.step_bound(GOLD["g_%s_%s" % (name, state)], W, k, 0.1)
    assert lo.within(GOLD["g_%s_step_%s" % (name, state)], new, alt, bound).all()
    assert np.isfinite(bound).all() and (bound > 0).all()


def _state(name="sensor300", state="run10"):
    W = _graph(name)
    return W, GOLD["g_%s_%s" % (name, state)], np.sqrt(1.0 / W.shape[0])


def test_bound_grows_where_forces_cancel():
    W, pos, k = _state()
    new, alt, bound = lo.step_bound(pos, W, k, 0.1)
    L = np.array([np.linalg.norm(lo.displacement(pos, W, k, i)) for i in range(W.shape[0])])
    big, small = np.argmax(L), np.argmin(L)
    assert bound[small].max() > 10 * bound[big].max()


def test_bound_rejects_a_dropped_neighbour():
    W, pos, k = _state()
    i = int(np.argmax(np.diff(W.indptr)))
    Wd = sparse.lil_matrix(W)
    Wd[i, W.indices[W.indptr[i]]] = 0
    got = lo.step(pos, sparse.csr_matrix(Wd), k, 0.1, rows=[i])
    new, alt, bound = lo.step_bound(pos, W, k, 0.1, rows=[i])
    assert not lo.within(got, new, alt, bound).any()


def test_bound_rejects_a_doubled_repulsion_term():
    W, pos, k = _state()
    i, j = 3, 150
    disp = lo.displacement(pos, W, k, i)
    delta = pos[i] - pos[j]
    d = max(np.sqrt((delta ** 2).sum()), 0.01)
    disp = disp + delta * k * k / d ** 2
    got = pos[i] + disp * 0.1 / max(np.linalg.norm(disp), 0.01)
    new, alt, bound = lo.step_bound(pos, W, k, 0.1, rows=[i])
    assert not lo.within(got[None], new, alt, bound).any()


def test_bound_rejects_the_wrong_length_branch_far_from_the_threshold():
    W, pos, k = _state()
    rows = np.arange(W.shape[0])
    new, alt, bound = lo.step_bound(pos, W, k, 0.1)
    disp = np.stack([lo.displacement(pos, W, k, i) for i in rows])
    L = np.linalg.norm(disp, axis=1)
    far = np.flatnonzero(L > 0.05)
    assert far.size
    wrong = pos[far] + disp[far] * 0.1 / 0.1
    assert not lo.within(wrong, new[far], alt[far], bound[far]).any()
    np.testing.assert_array_equal(alt[far], new[far])


def test_fixed_vertices_have_zero_bound():
    W, pos, k = _state()
    new, alt, bound = lo.step_bound(pos, W, k, 0.1, fixed=[2, 7])
    assert (bound[[2, 7]] == 0).all()
    np.testing.assert_array_equal(new[[2, 7]], pos[[2, 7]])
