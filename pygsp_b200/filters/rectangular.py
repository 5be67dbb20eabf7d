"""Rectangular filter (mirror of pygsp/filters/rectangular.py:53-83)."""
import numpy as np

from .filter import Filter


class Rectangular(Filter):
    r"""Ideal band-pass: 1 where ``band_min <= x / lmax <= band_max``, 0 elsewhere.

    A bound of None leaves that side open (low- or high-pass); with neither bound the filter is
    1.  ``G.lmax`` is read when the kernel is evaluated, as in the reference.
    """

    def __init__(self, G, band_min=None, band_max=0.2):
        self.band_min = band_min
        self.band_max = band_max

        def lowpass(x):
            return np.asanyarray(x) / G.lmax <= band_max

        def highpass(x):
            return np.asanyarray(x) / G.lmax >= band_min

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
        return attrs
