"""oracle/filter_banks_oracle.py against the unmodified PyGSP 0.6.1 (tests/golden/filter_banks.npz).

Given the reference's own basis (e, U), the restatements of Gabor and Modulation (both orders)
reproduce the reference's outputs, signs included.  CPU only."""
import numpy as np
import pytest

from conftest import csr_from
from oracle import filter_banks_oracle as fbo
from oracle import pygsp_oracle as orc


@pytest.fixture(scope="module")
def gold(golden):
    return golden("filter_banks")


def _rect(lmax, band_min, band_max):
    def kernel(x):
        x = np.asarray(x) / lmax
        y = x <= band_max
        if band_min is not None:
            y = y & (x >= band_min)
        return y.astype(np.float64)
    return kernel


def test_gabor(gold):
    lmax, e, U, s = float(gold["lmax"]), gold["e"], gold["U"], gold["signal"]
    np.testing.assert_allclose(fbo.gabor(e, U, _rect(lmax, None, 0.1), s), gold["gabor_rect"],
                               atol=1e-12)
    np.testing.assert_allclose(fbo.gabor(e, U, _rect(lmax, 0, 0), s), gold["gabor_delta"],
                               atol=1e-12)


def test_modulation_first(gold):
    lmax, e, U, s = float(gold["lmax"]), gold["e"], gold["U"], gold["signal"]
    for name, k in (("delta", _rect(lmax, 0, 0)), ("rect", _rect(lmax, None, 0.1))):
        np.testing.assert_allclose(fbo.modulation_first(e, U, k(e), s),
                                   gold["mod_first_" + name], atol=1e-12)


def test_windowed_gft(golden, gold):
    lmax, U, s = float(gold["lmax"]), gold["U"], gold["signal"]
    n = U.shape[0]
    L = orc.laplacian(csr_from(golden("sensor123"), "W").astype(np.float64))
    windows = orc.filter_signal(L, lmax, [_rect(lmax, None, 0.1)], np.identity(n)) * np.sqrt(n)
    np.testing.assert_allclose(fbo.windowed_gft(U, windows, s), gold["mod_second_rect"],
                               atol=1e-11)
