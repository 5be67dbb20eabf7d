"""Exponential window filter (mirror of pygsp/filters/expwin.py:53-84)."""
import numpy as np

from .filter import Filter


def _ramp(x, slope):
    """exp(-slope / x) for x > 0, 0 elsewhere: smooth, and flat to every order at 0."""
    x = np.asanyarray(x, dtype=np.float64)
    positive = x > 0
    return np.where(positive, np.exp(-slope / np.where(positive, x, 1.0)), 0.0)


def _step(x, slope):
    """Smooth step from 0 (x <= 0) to 1 (x >= 1)."""
    up, down = _ramp(x, slope), _ramp(1 - np.asanyarray(x, dtype=np.float64), slope)
    return up / (up + down)


class Expwin(Filter):
    r"""Smooth band-pass (or low- / high-pass) window on [band_min, band_max] (in units of lmax).

    The edges are the smooth step ``h(t) = e(t) / (e(t) + e(1 - t))``, ``e(t) = exp(-slope / t)``:
    low-pass ``h(1/2 - x/lmax + band_max)``, high-pass ``h(1/2 + x/lmax - band_min)``, their
    product for a band; with neither bound the filter is 1.  ``G.lmax`` is read when the kernel is
    evaluated, as in the reference.
    """

    def __init__(self, G, band_min=None, band_max=0.2, slope=1):
        self.band_min = band_min
        self.band_max = band_max
        self.slope = slope

        def lowpass(x):
            return _step(0.5 - np.asanyarray(x) / G.lmax + band_max, slope)

        def highpass(x):
            return _step(0.5 + np.asanyarray(x) / G.lmax - band_min, slope)

        if band_min is None and band_max is None:
            kernel = np.ones_like
        elif band_min is None:
            kernel = lowpass
        elif band_max is None:
            kernel = highpass
        else:
            def kernel(x):
                return lowpass(x) * highpass(x)
        super().__init__(G, kernel)

    def _get_extra_repr(self):
        attrs = dict()
        if self.band_min is not None:
            attrs["band_min"] = "{:.2f}".format(self.band_min)
        if self.band_max is not None:
            attrs["band_max"] = "{:.2f}".format(self.band_max)
        attrs["slope"] = "{:.0f}".format(self.slope)
        return attrs
