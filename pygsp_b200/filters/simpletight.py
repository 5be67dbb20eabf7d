"""Simple tight frame (mirror of pygsp/filters/simpletight.py:49-97)."""
import numpy as np

from .filter import Filter


def _h(t):
    return np.sin(np.pi * t / 2.0) ** 2


def _simple_tight(x, wavelet):
    r"""Scaling function (1 below 1/4, ``sqrt(1 - h(4x - 1)^2)`` on [1/4, 1/2)) or wavelet
    (``h(4x - 1)`` on [1/4, 1/2), ``sqrt(1 - h(2x - 1)^2)`` on [1/2, 1)), ``h(t) = sin(pi t / 2)^2``."""
    x = np.asanyarray(x, dtype=np.float64)
    rise = (x >= 0.25) & (x < 0.5)
    fall = (x >= 0.5) & (x < 1.0)
    y = np.zeros(x.shape)
    if wavelet:
        y[rise] = _h(4 * (x[rise] - 0.25))
        y[fall] = np.sqrt(1 - _h(2 * x[fall] - 1) ** 2)
    else:
        y[x < 0.25] = 1.0
        y[rise] = np.sqrt(1 - _h(4 * x[rise] - 1) ** 2)
    return y


class SimpleTight(Filter):
    r"""A tight frame of one scaling function and ``Nf - 1`` wavelets with simple transitions.

    Filter 0 is the scaling function at ``scales[0] x``, filter i + 1 the wavelet at
    ``scales[i] x``.  The default scales ``2^(Nf-2) / (2 lmax) .. 1 / (2 lmax)`` are frozen from
    ``G.lmax`` at construction (an empty ``scales`` also takes them); ``len(scales)`` must be
    ``Nf - 1``.
    """

    def __init__(self, G, Nf=6, scales=None):
        if scales is None or len(scales) == 0:
            scales = 1.0 / (2.0 * G.lmax) * np.power(2, np.arange(Nf - 2, -1, -1))
        self.scales = scales
        if len(scales) != Nf - 1:
            raise ValueError("len(scales) should be Nf-1.")
        kernels = [lambda x: _simple_tight(scales[0] * np.asanyarray(x), wavelet=False)]
        kernels += [lambda x, i=i: _simple_tight(scales[i] * np.asanyarray(x), wavelet=True)
                    for i in range(Nf - 1)]
        super().__init__(G, kernels)
