"""Held's tight frame (mirror of pygsp/filters/held.py:44-74)."""
import numpy as np

from .tight import TightPair, piecewise_lowpass


class Held(TightPair):
    r"""Held's low-pass and its complement: a tight frame of two filters.

    On ``y = 2 x / lmax`` the low-pass is 1 below ``a``, ``sin(2 pi mu(y / (8 a)))`` on
    [a, 2a) with ``mu(t) = -1 + 24 t - 144 t^2 + 256 t^3``, and 0 from 2a on.
    """

    def __init__(self, G, a=2.0 / 3):
        self.a = a

        def mu(t):
            return -1 + 24 * t - 144 * t ** 2 + 256 * t ** 3

        super().__init__(G, lambda y: piecewise_lowpass(
            y, a, 2 * a, lambda t: np.sin(2 * np.pi * mu(t / 8 / a))))

    def _get_extra_repr(self):
        return dict(a="{:.2f}".format(self.a))
