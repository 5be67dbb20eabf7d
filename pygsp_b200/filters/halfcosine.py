"""Half-cosine filter bank (mirror of pygsp/filters/halfcosine.py:34-52)."""
import numpy as np

from .filter import Filter


class HalfCosine(Filter):
    r"""``Nf`` raised-cosine bumps, uniformly translated over [0, lmax].

    The bump is ``(1 + cos(2 pi (x / d - 1/2))) / 2`` on [0, d], ``d = 3 lmax / (Nf - 2)``, and
    filter i is the bump shifted by ``d (i - 2) / 3``; the squares sum to a constant over most of
    the spectrum.  ``d`` is frozen from ``G.lmax`` at construction.
    """

    def __init__(self, G, Nf=6):
        if Nf <= 2:
            raise ValueError("The number of filters must be greater than 2.")
        width = G.lmax * 3 / (Nf - 2)

        def bump(x):
            y = 0.5 + 0.5 * np.cos(2 * np.pi * (x / width - 0.5))
            return y * (x >= 0) * (x <= width)

        kernels = [lambda x, i=i: bump(np.asanyarray(x) - width / 3 * (i - 2)) for i in range(Nf)]
        super().__init__(G, kernels)
