"""Simoncelli's tight frame (mirror of pygsp/filters/simoncelli.py:38-67)."""
import numpy as np

from .tight import TightPair, piecewise_lowpass


class Simoncelli(TightPair):
    r"""Simoncelli's low-pass and its complement: a tight frame of two filters.

    On ``y = 2 x / lmax`` the low-pass is 1 below ``a``, ``cos(pi/2 log2(y / a))`` on [a, 2a),
    and 0 from 2a on.
    """

    def __init__(self, G, a=2 / 3):
        self.a = a
        super().__init__(G, lambda y: piecewise_lowpass(
            y, a, 2 * a, lambda t: np.cos(np.pi / 2 * np.log(t / a) / np.log(2))))

    def _get_extra_repr(self):
        return dict(a="{:.2f}".format(self.a))
