"""Papadakis's tight frame (mirror of pygsp/filters/papadakis.py:38-67)."""
import numpy as np

from .tight import TightPair, piecewise_lowpass


class Papadakis(TightPair):
    r"""Papadakis's low-pass and its complement: a tight frame of two filters.

    On ``y = 2 x / lmax`` the low-pass is 1 below ``a``, ``sqrt((1 - sin(3 pi y / (2 a))) / 2)``
    on [a, 5a/3), and 0 from 5a/3 on.
    """

    def __init__(self, G, a=0.75):
        self.a = a
        super().__init__(G, lambda y: piecewise_lowpass(
            y, a, a * 5 / 3, lambda t: np.sqrt((1 - np.sin(3 * np.pi / (2 * a) * t)) / 2)))

    def _get_extra_repr(self):
        return dict(a="{:.2f}".format(self.a))
