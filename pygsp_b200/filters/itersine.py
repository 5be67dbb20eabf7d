"""Iterated-sine filter bank (mirror of pygsp/filters/itersine.py:34-60)."""
import numpy as np

from .filter import Filter


class Itersine(Filter):
    r"""``Nf`` translates of the iterated sine ``sin(pi/2 cos(pi t)^2)`` on |t| <= 1/2.

    Filter i (1-based) is ``sqrt(2 / overlap) k(x / s - (i - overlap/2) / overlap)`` with
    ``s = overlap lmax / (Nf - overlap + 1)``: a tight frame.  ``s`` and the centres ``mu`` are
    frozen from ``G.lmax`` at construction.
    """

    def __init__(self, G, Nf=6, overlap=2):
        self.overlap = overlap
        self.mu = np.linspace(0, G.lmax, num=Nf)
        scale = G.lmax / (Nf - overlap + 1) * overlap
        gain = np.sqrt(2 / overlap)

        def bump(t):
            y = np.sin(0.5 * np.pi * np.cos(t * np.pi) ** 2)
            return y * ((t >= -0.5) * (t <= 0.5))

        kernels = [lambda x, i=i: gain * bump(np.asanyarray(x) / scale - (i - overlap / 2) / overlap)
                   for i in range(1, Nf + 1)]
        super().__init__(G, kernels)

    def _get_extra_repr(self):
        return dict(overlap="{:.2f}".format(self.overlap))
