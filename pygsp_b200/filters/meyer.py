"""Meyer wavelet bank (mirror of pygsp/filters/meyer.py:45-89)."""
import numpy as np

from .filter import Filter

_L1, _L2, _L3 = 2 / 3.0, 4 / 3.0, 8 / 3.0


def _nu(t):
    """Meyer's auxiliary polynomial: 0 at t = 0, 1 at t = 1, flat to third order at both ends."""
    return t ** 4 * (35 - 84 * t + 70 * t ** 2 - 20 * t ** 3)


def _meyer(x, wavelet):
    r"""Scaling function (1 below 2/3, a cosine roll-off to 4/3) or wavelet (a sine rise on
    [2/3, 4/3), a cosine fall on [4/3, 8/3)) of the Meyer frame."""
    x = np.asanyarray(x, dtype=np.float64)
    rise = (x >= _L1) & (x < _L2)
    fall = (x >= _L2) & (x < _L3)
    y = np.zeros(x.shape)
    if wavelet:
        y[rise] = np.sin(np.pi / 2 * _nu(np.abs(x[rise]) / _L1 - 1))
        y[fall] = np.cos(np.pi / 2 * _nu(np.abs(x[fall]) / _L2 - 1))
    else:
        y[x < _L1] = 1
        y[rise] = np.cos(np.pi / 2 * _nu(np.abs(x[rise]) / _L1 - 1))
    return y


class Meyer(Filter):
    r"""Meyer's tight frame: one scaling function and ``Nf - 1`` wavelets.

    Filter 0 is the scaling function at ``scales[0] x``, filter i + 1 the wavelet at
    ``scales[i] x``.  The default scales ``4 / (3 lmax) 2^(Nf-2) .. 4 / (3 lmax)`` are frozen from
    ``G.lmax`` at construction; ``len(scales)`` must be ``Nf - 1``.
    """

    def __init__(self, G, Nf=6, scales=None):
        if scales is None:
            scales = (4.0 / (3 * G.lmax)) * np.power(2.0, np.arange(Nf - 2, -1, -1))
        self.scales = scales
        if len(scales) != Nf - 1:
            raise ValueError("len(scales) should be Nf-1.")
        kernels = [lambda x: _meyer(scales[0] * np.asanyarray(x), wavelet=False)]
        kernels += [lambda x, i=i: _meyer(scales[i] * np.asanyarray(x), wavelet=True)
                    for i in range(Nf - 1)]
        super().__init__(G, kernels)
