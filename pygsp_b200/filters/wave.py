"""Wave equation filter bank (mirror of pygsp/filters/wave.py:86-128)."""
import numpy as np

from .filter import Filter


def _as_list(v):
    try:
        return list(v)
    except TypeError:
        return [v]


class Wave(Filter):
    r"""Solutions of the graph wave equation: ``g(x) = cos(t arccos(1 - s^2 x / (2 lmax)))``.

    One filter per (time t, speed s) pair.  A scalar (or one-element) ``time`` or ``speed`` is
    repeated to the other's length; two lists must have the same length.  The speed must lie in
    [0, 2[, where the argument of arccos stays in [-1, 1].  ``G.lmax`` is read when the kernel is
    evaluated, as in the reference.
    """

    def __init__(self, G, time=10, speed=1):
        time, speed = _as_list(time), _as_list(speed)
        self.time = time
        self.speed = speed
        if len(time) != len(speed):
            if len(speed) == 1:
                speed = speed * len(time)
            elif len(time) == 1:
                time = time * len(speed)
            else:
                raise ValueError("If both parameters are iterable, "
                                 "they should have the same length.")
        if np.any(np.asanyarray(speed) >= 2):
            raise ValueError("The wave propagation speed should be in [0, 2[")

        def kernel(x, t, s):
            return np.cos(t * np.arccos(1 - s ** 2 * np.asanyarray(x) / G.lmax / 2))

        super().__init__(G, [lambda x, t=t, s=s: kernel(x, t, s) for t, s in zip(time, speed)])

    def _get_extra_repr(self):
        time = "[" + ", ".join("{:.2f}".format(t) for t in self.time) + "]"
        speed = "[" + ", ".join("{:.2f}".format(s) for s in self.speed) + "]"
        return dict(time=time, speed=speed)
