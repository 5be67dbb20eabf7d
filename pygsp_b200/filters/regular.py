"""Regular tight frame (mirror of pygsp/filters/regular.py:46-66)."""
import numpy as np

from .tight import TightPair


class Regular(TightPair):
    r"""A low-pass of chosen smoothness and its complement: a tight frame of two filters.

    On ``y = 2 x / lmax``: ``degree = 0`` gives ``sin(pi y / 4)``; otherwise
    ``s = sin(pi (y - 1) / 2)`` is passed ``degree - 2`` more times through ``s -> sin(pi s / 2)``
    and the low-pass is ``sin(pi (1 + s) / 4)``.  A higher degree gives a smoother filter.
    """

    def __init__(self, G, degree=3):
        self.degree = degree

        def lowpass(y):
            if degree == 0:
                return np.sin(np.pi / 4 * y)
            s = np.sin(np.pi * (y - 1) / 2)
            for _ in range(degree - 2):
                s = np.sin(np.pi * s / 2)
            return np.sin(np.pi / 4 * (1 + s))

        super().__init__(G, lowpass)
