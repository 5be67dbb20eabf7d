"""Shared part of the two-filter tight frames Held, Papadakis, Regular and Simoncelli.

Each of them is a low-pass ``h(2 x / lmax)`` and its complement ``sqrt(1 - h^2)`` (the
reference's ``complement(frame_bound=1)``), so that the squares of the two sum to 1.
"""
import numpy as np

from .filter import Filter


def piecewise_lowpass(y, edge, stop, roll):
    """1 on [0, edge), ``roll(y)`` on [edge, stop), 0 from stop on (and below 0)."""
    y = np.asanyarray(y, dtype=np.float64)
    out = np.zeros(y.shape)
    out[(y >= 0) & (y < edge)] = 1
    band = (y >= edge) & (y < stop)
    out[band] = roll(y[band])
    return out


class TightPair(Filter):
    """A low-pass ``h(2 x / lmax)`` and its complement to a tight frame of bound 1."""

    def __init__(self, G, h):
        lowpass = Filter(G, lambda x: h(np.asanyarray(x) * 2 / G.lmax))
        super().__init__(G, lowpass._kernels + lowpass.complement(frame_bound=1)._kernels)
