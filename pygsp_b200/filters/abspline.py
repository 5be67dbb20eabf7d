"""Abspline wavelet bank (mirror of pygsp/filters/abspline.py:64-111)."""
import numpy as np
from scipy import optimize

from .. import utils
from .filter import Filter


def _abspline(x, alpha=2, beta=2, t1=1.0, t2=2.0):
    r"""``(x / t1)^alpha`` below t1, ``(t2 / x)^beta`` from t2 on, and between them the cubic that
    meets both pieces with matching values (1) and slopes (alpha / t1, -beta / t2)."""
    x = np.asanyarray(x, dtype=np.float64)
    # Hermite conditions on a0 + a1 x + a2 x^2 + a3 x^3: values at t1, t2, slopes at t1, t2
    system = np.array([[1, t1, t1 ** 2, t1 ** 3],
                       [1, t2, t2 ** 2, t2 ** 3],
                       [0, 1, 2 * t1, 3 * t1 ** 2],
                       [0, 1, 2 * t2, 3 * t2 ** 2]], dtype=np.float64)
    a = np.linalg.solve(system, np.array([1.0, 1.0, alpha / t1, -beta / t2]))
    low, high = x <= t1, x >= t2
    mid = (x >= t1) & (x < t2)
    y = np.zeros(x.shape)
    y[low] = x[low] ** alpha * t1 ** (-alpha)
    xm = x[mid]
    y[mid] = a[0] + a[1] * xm + a[2] * xm ** 2 + a[3] * xm ** 3
    y[high] = x[high] ** (-beta) * t2 ** beta
    return y


class Abspline(Filter):
    r"""One low-pass plus ``Nf - 1`` band-pass "abspline" wavelets.

    The band-pass ``g(t x)`` is monic ``x^2`` below 1, ``4 / x^2`` above 2 and a cubic spline in
    between; the scales ``t_i`` are log-spaced between ``2/lmin`` and ``1/lmax`` (``lmin = lmax /
    lpfactor``).  The low-pass is ``gamma exp(-(x / (0.6 lmin))^4)`` with ``gamma`` the peak of
    the band-pass on [1, 2], found by bounded scalar minimisation as in the reference.  ``lmin``
    and the scales are frozen from ``G.lmax`` at construction.
    """

    def __init__(self, G, Nf=6, lpfactor=20, scales=None):
        self.lpfactor = lpfactor
        lmin = G.lmax / lpfactor
        if scales is None:
            scales = utils.compute_log_scales(lmin, G.lmax, Nf - 1)
        self.scales = scales
        peak = optimize.minimize_scalar(lambda t: -_abspline(t), bounds=(1, 2), method="bounded")
        gamma = float(_abspline(peak.x))
        width = 0.6 * lmin

        def lowpass(x):
            return gamma * np.exp(-np.power(np.asanyarray(x) / width, 4))

        kernels = [lowpass] + [lambda x, i=i: _abspline(self.scales[i] * np.asanyarray(x))
                               for i in range(Nf - 1)]
        super().__init__(G, kernels)

    def _get_extra_repr(self):
        return dict(lpfactor="{:.2f}".format(self.lpfactor))
