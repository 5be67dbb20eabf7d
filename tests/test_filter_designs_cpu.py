"""The filter designs and the frame methods of Filter on the host, against the unmodified PyGSP
0.6.1 (tests/golden/filter_banks.npz, made by tests/golden/make_golden_filter_banks.py).

Everything here is host NumPy on the responses: the graph is a stand-in object holding only
lmax, e and N, so no device is needed.  Checks ported from the reference's test_filters.py are
restated in this file's own words."""
import importlib.util
import logging
import os

import numpy as np
import pytest

from conftest import GOLDEN

from pygsp_b200 import filters

TOL = 1e-12


def _designs():
    spec = importlib.util.spec_from_file_location(
        "make_golden_filter_banks", os.path.join(GOLDEN, "make_golden_filter_banks.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.DESIGNS


DESIGNS = _designs()
CASES = [(name, cls, kwargs) for name, (cls, default, alt) in DESIGNS.items()
         for name, kwargs in ((name, default), (name + "_alt", alt))]


class StandIn:
    """The part of a graph the designs read: lmax, the eigenvalues and the vertex count."""

    def __init__(self, lmax, e):
        self.lmax, self.e, self.N = float(lmax), np.asarray(e), len(e)


@pytest.fixture(scope="module")
def gold(golden):
    return golden("filter_banks")


@pytest.fixture(scope="module")
def G(gold):
    return StandIn(gold["lmax"], gold["e"])


@pytest.mark.parametrize("name,cls,kwargs", CASES, ids=[c[0] for c in CASES])
def test_design_responses_and_bounds(gold, G, name, cls, kwargs):
    f = getattr(filters, cls)(G, **kwargs)
    assert f.Nf == gold[name + "_e"].shape[0]
    np.testing.assert_allclose(f.evaluate(gold["grid"]), gold[name + "_grid"], rtol=TOL, atol=TOL)
    np.testing.assert_allclose(f.evaluate(G.e), gold[name + "_e"], rtol=TOL, atol=TOL)
    np.testing.assert_allclose(f.estimate_frame_bounds(), gold[name + "_bounds"], rtol=TOL,
                               atol=TOL)
    # the response keeps the shape of its argument
    assert f.evaluate(np.full((2, 3), 0.5 * G.lmax)).shape == (f.Nf, 2, 3)


def _banks(G):
    return {"heat234": filters.Heat(G, scale=[2, 3, 4]), "abspline5": filters.Abspline(G, 5),
            "expwin": filters.Expwin(G)}


@pytest.mark.parametrize("name", ["heat234", "abspline5", "expwin"])
def test_complement_and_inverse(gold, G, name):
    g = _banks(G)[name]
    c = g.complement(2.5)
    assert c.Nf == 1
    for where, x in (("grid", gold["grid"]), ("e", G.e)):
        if name + "_compl_raises" in gold:
            with pytest.raises(ValueError, match="not feasible"):
                c.evaluate(x)
        else:
            np.testing.assert_allclose(c.evaluate(x), gold[name + "_compl_" + where], rtol=TOL,
                                       atol=TOL)
        # the inverse of a bank that is not a frame is 1/g where g is tiny: compare relatively
        h = g.inverse()
        assert h.Nf == g.Nf
        np.testing.assert_allclose(h.evaluate(x), gold[name + "_inv_" + where], rtol=TOL, atol=TOL)


def test_frame_bounds_of_simple_banks(G):
    # an ideal low-pass has a null space (A = 0); a constant 2 is a tight frame of bound 4
    assert filters.Rectangular(G).estimate_frame_bounds() == (0, 1)
    assert filters.Filter(G, lambda x: np.full_like(x, 2)).estimate_frame_bounds() == (4, 4)
    A, B = filters.Heat(G, 10).estimate_frame_bounds(G.e)
    assert A == pytest.approx(np.exp(-10 * G.e[-1] / G.lmax) ** 2) and B == 1


def test_complement_makes_a_tight_frame(G):
    g = filters.MexicanHat(G)
    tight = g + g.complement(2.5)
    np.testing.assert_allclose(tight.estimate_frame_bounds(), (2.5, 2.5), rtol=1e-12)
    # with no bound, the complement reaches the largest energy of the frequencies it is given
    tight = g + g.complement()
    A, B = tight.estimate_frame_bounds()
    assert A == pytest.approx(B, rel=1e-12)
    with pytest.raises(ValueError, match="Choose at least"):
        g.complement(0.1).evaluate(np.array([0.0, 1.0]))


def test_inverse_of_a_tight_frame_is_the_bank_over_its_bound(G):
    g = filters.Expwin(G)
    g = g + g.complement(3)
    h = g.inverse()
    np.testing.assert_allclose(h.evaluate(G.e), g.evaluate(G.e) / 3, atol=1e-10)
    A, B = filters.Heat(G, scale=[2, 3, 4]).estimate_frame_bounds()
    Ah, Bh = filters.Heat(G, scale=[2, 3, 4]).inverse().estimate_frame_bounds()
    assert A * Bh == pytest.approx(1, rel=1e-10) and B * Ah == pytest.approx(1, rel=1e-10)


def test_inverse_logs(G, caplog):
    with caplog.at_level(logging.WARNING):
        h = filters.Expwin(G).inverse()
    assert any("not invertible" in r.getMessage() for r in caplog.records)
    assert np.all(h.evaluate(np.array([G.lmax])) == 0)        # zero where every response is 0
    caplog.clear()
    with caplog.at_level(logging.WARNING):
        filters.Heat(G, scale=[40]).inverse()                  # A / B = exp(-80) < 1e-10
    assert any("badly conditioned" in r.getMessage() for r in caplog.records)
    caplog.clear()
    with caplog.at_level(logging.WARNING):
        filters.Meyer(G).inverse()
    assert not caplog.records


def test_value_errors(G):
    with pytest.raises(ValueError):
        filters.HalfCosine(G, Nf=2)
    with pytest.raises(ValueError):
        filters.Meyer(G, Nf=4, scales=[1.0, 2.0])
    with pytest.raises(ValueError):
        filters.SimpleTight(G, Nf=4, scales=[1.0, 2.0])
    with pytest.raises(ValueError):
        filters.MexicanHat(G, Nf=4, scales=[1.0, 2.0])
    with pytest.raises(ValueError, match="speed"):
        filters.Wave(G, speed=2)
    with pytest.raises(ValueError, match="speed"):
        filters.Wave(G, time=[1, 2], speed=[0.5, 2.5])
    with pytest.raises(ValueError, match="same length"):
        filters.Wave(G, time=[1, 2, 3], speed=[0.5, 1.0])
    other = StandIn(G.lmax, G.e)
    for bank in (filters.Gabor, filters.Modulation):
        with pytest.raises(ValueError, match="one filter"):
            bank(G, filters.Regular(G))
        with pytest.raises(ValueError, match="mother kernel"):
            bank(G, filters.Rectangular(other, None, 0.1))


def test_wave_broadcasting(G):
    assert filters.Wave(G, time=[1, 2, 3], speed=1).Nf == 3
    assert filters.Wave(G, time=4, speed=[0.5, 1.0]).Nf == 2
    w = filters.Wave(G, time=[1, 2], speed=[0.5, 1.5])
    x = np.linspace(0, G.lmax, 5)
    np.testing.assert_allclose(w.evaluate(x)[1],
                               np.cos(2 * np.arccos(1 - 1.5 ** 2 * x / G.lmax / 2)), rtol=1e-15)
    assert repr(w) == "Wave(in=1, out=2, time=[1.00, 2.00], speed=[0.50, 1.50])"


def test_scales_are_frozen_at_construction(G):
    lmax = G.lmax
    g = filters.Meyer(G)
    before = g.evaluate(G.e)
    G.lmax = 2 * lmax
    try:
        np.testing.assert_array_equal(g.evaluate(G.e), before)
    finally:
        G.lmax = lmax


def test_gabor_translates_the_kernel(G):
    k = filters.Heat(G, 5)
    g = filters.Gabor(G, k)
    assert g.Nf == G.N
    x = np.linspace(0, G.lmax, 7)
    np.testing.assert_array_equal(g.evaluate(x)[17], k.evaluate(x - G.e[17])[0])


def test_reprs(G):
    assert repr(filters.Expwin(G)) == "Expwin(in=1, out=1, band_max=0.20, slope=1)"
    assert repr(filters.Rectangular(G, 0.1, None)) == "Rectangular(in=1, out=1, band_min=0.10)"
    assert repr(filters.Abspline(G)) == "Abspline(in=1, out=6, lpfactor=20.00)"
    assert repr(filters.Held(G)) == "Held(in=1, out=2, a=0.67)"
    assert repr(filters.Itersine(G)) == "Itersine(in=1, out=6, overlap=2.00)"
    assert repr(filters.Meyer(G)) == "Meyer(in=1, out=6)"
