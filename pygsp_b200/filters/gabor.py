"""Gabor filter bank (mirror of pygsp/filters/gabor.py:56-92)."""
import numpy as np

from .filter import Filter


def check_mother_kernel(graph, kernel):
    """A Gabor-type bank is built from ONE filter defined on the same graph object."""
    if kernel.n_filters != 1:
        raise ValueError("A kernel must be one filter. The passed "
                         "filter bank {} has {}.".format(kernel, kernel.n_filters))
    if kernel.G is not graph:
        raise ValueError("The graph passed to this filter bank must "
                         "be the one used to build the mother kernel.")


class Gabor(Filter):
    r"""The mother kernel ``g`` translated to every graph frequency: ``g_i(x) = g(x - e_i)``.

    One filter per vertex (``N`` filters); the eigenvalues ``G.e`` are read when a kernel is
    evaluated.  :meth:`filter` always filters exactly through the Fourier basis, as the reference
    does: the translated responses have no short Chebyshev expansion.
    """

    def __init__(self, graph, kernel):
        check_mother_kernel(graph, kernel)
        kernels = [lambda x, i=i: kernel.evaluate(np.asanyarray(x) - graph.e[i])[0]
                   for i in range(graph.N)]
        super().__init__(graph, kernels)

    def filter(self, s, method="exact", order=None):
        r"""Filter ``s`` exactly (``method`` and ``order`` are ignored, filter.py / gabor.py:90)."""
        return super().filter(s, method="exact")
