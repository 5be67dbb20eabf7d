"""pygsp_b200 -- Hopper-native Chebyshev spectral graph filtering.

Drop-in for the ``Graph.compute_laplacian`` -> ``Graph.estimate_lmax`` ->
``Filter.filter(method='chebyshev')`` -> ``approximations.cheby_op`` path of
PyGSP 0.6.1, computed by hand-written sm_90a CUDA kernels (``libgspb200.so``)
behind the reference's Python API.  There is no CPU fallback.
"""
from . import _native  # noqa: F401
from . import utils  # noqa: F401
from . import graphs  # noqa: F401
from . import filters  # noqa: F401
from . import reduction  # noqa: F401
from . import learning  # noqa: F401
from . import features  # noqa: F401
from . import optimization  # noqa: F401

__version__ = "0.1.0"


def patch_pygsp(dtype=None):
    """Route the *reference's* ``Filter.filter`` through this engine.

    ``pygsp.filters.filter`` looks ``approximations.cheby_op`` up on the module at
    call time (filter.py:309,319), so rebinding it is enough: a stock
    ``pygsp.graphs.Graph`` then has its Laplacian uploaded once and every Chebyshev
    recurrence runs on the GPU.  ``dtype`` (torch.float32 default, torch.float64 for the
    reference's own test tolerances) is the engine type for graphs that do not set
    ``G._gspb200_dtype`` themselves.  Returns the original function; ``unpatch_pygsp()``
    restores it.
    """
    import pygsp.filters.approximations as ref
    from .filters import approximations as ours
    if dtype is not None:
        ours.PATCH_DEFAULT_DTYPE = dtype
    ref._cheby_op_scipy = getattr(ref, "_cheby_op_scipy", ref.cheby_op)
    ref.cheby_op = ours.cheby_op
    return ref._cheby_op_scipy


def unpatch_pygsp():
    import pygsp.filters.approximations as ref
    if hasattr(ref, "_cheby_op_scipy"):
        ref.cheby_op = ref._cheby_op_scipy
