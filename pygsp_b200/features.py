r"""Graph features on the device: mirror of ``pygsp/features.py``.

``compute_norm_tig`` and ``compute_spectrogram`` need the squared row norms of the frame
``||p(L) e_i||^2``, which the reference gets by filtering the identity: an N Nf x N matrix per
kernel, and M of them for a spectrogram (features.py:41, 58, 88-91).  Here no frame is built.
The reference filters with the order-m Chebyshev approximant ``p = c0/2 T_0 + sum_k c_k T_k(Lt)``
(approximations.py:58-114), so for a symmetric L

    ||p(L) e_i||^2 = e_i^T p(L)^2 e_i = sum_{n <= 2m} d_n mu_n(i),   mu_n(i) = (T_n(Lt))_ii,

with d the exact Chebyshev series of p^2 (:func:`~pygsp_b200.filters.approximations.
cheby_square_coeff`).  One recurrence over identity probe blocks gives the moments mu
(:func:`~pygsp_b200.filters.approximations.cheby_moments_device`, csrc/moments.cu); every kernel
of a bank and every atom of a spectrogram is then one column of ``mu D^T``, formed in one pass by
``gsp_block_combine_f64``.  ``compute_avg_adj_deg`` counts the entries of the boolean product
``A A`` on the device (``gsp_two_hop_count_*``).
"""
import numpy as np

from . import _native as nat
from . import utils
from .filters import approximations
from .filters.filter import Filter

_logger = utils.build_logger(__name__)


def compute_avg_adj_deg(G):
    r"""Average adjacency degree of every vertex (features.py:11-23).

    ``sum(A A, axis=1) / (sum(A, axis=1) + 1)`` with ``A = W > 0`` (graph.py:718-727).  The
    product of boolean matrices is a logical OR, so the numerator is the number of *distinct*
    vertices at the end of a walk of exactly two steps; the denominator is the out-degree plus
    one.  Returns a float64 ndarray of shape (N, 1) (the reference returns an ``np.matrix``).
    """
    from .graphs.csr import DeviceCSR
    torch = nat.require_cuda()
    W = G.W
    if not isinstance(W, DeviceCSR):                      # a reference graph: upload W once
        from scipy import sparse
        dev = torch.device("cuda:%d" % torch.cuda.current_device())
        W = DeviceCSR.from_scipy(sparse.csr_matrix(W), torch.float64, dev)
    n = W.shape[0]
    two_hop = torch.empty(n, dtype=torch.int32, device=W.device)
    degree = torch.empty(n, dtype=torch.int32, device=W.device)
    with torch.cuda.device(W.device):
        nat.call("gsp_two_hop_count_" + nat.suffix(W.dtype), nat.i64(n), W.indptr, W.indices,
                 W.data, two_hop, degree, nat.stream_ptr(W.device))
    num = two_hop.cpu().numpy().astype(np.float64)
    den = degree.cpu().numpy().astype(np.float64) + 1.0
    return (num / den).reshape(n, 1)


@utils.filterbank_handler
def compute_tig(g, **kwargs):
    r"""The frame of ``g``: ``g.compute_frame()`` (features.py:26-41), an (N Nf, N) ndarray.

    ``method`` and ``order`` are passed to the filtering (the reference drops every keyword).
    For a bank, the list of Nf copies that the reference's ``filterbank_handler`` returns.
    """
    kwargs.pop("i", None)
    return g.compute_frame(**kwargs)


def _square_norms(G, kernels, method="chebyshev", order=30):
    """(N, len(kernels)) float64 device tensor of ||k(L) e_i||^2 for every kernel k."""
    from .graphs import fourier
    torch = nat.require_cuda()
    if method == "exact":
        # filter.py:292-301 with s = I: ||U diag(k(e)) U^T e_i||^2 = sum_n U[i, n]^2 k(e_n)^2
        e = G.e
        resp = np.stack([np.asarray(k(e), dtype=np.float64) for k in kernels], axis=1)
        assert resp.shape[0] == G.N, "method='exact' needs the full Fourier basis"
        U = G._device_basis().to(torch.float64)
        return fourier.block_combine((U * U).contiguous(), resp ** 2)
    if method != "chebyshev":
        raise ValueError("Unknown method {}.".format(method))
    L = approximations._laplacian_on_device(G)
    lmax = G.lmax
    c = np.stack([approximations.compute_cheby_coeff(Filter(G, k), m=order) for k in kernels])
    d = approximations.cheby_square_coeff(c)                 # (nk, 2 order + 1)
    d[:, 0] *= 0.5                                           # the T_0 weight is d0 / 2
    mu = approximations.cheby_moments_device(L, lmax, order)
    return fourier.block_combine(mu, np.ascontiguousarray(d.T))


@utils.filterbank_handler
def compute_norm_tig(g, **kwargs):
    r"""l2 norm of every row of the frame of ``g`` (features.py:44-59), without the frame.

    Entry ``f N + j`` is ``||p_f(L) e_j||``, (N Nf,) float64; for a bank, a list of Nf copies
    (the reference's ``compute_frame`` ignores the filter index).  ``order`` (default 30, the
    reference's) is the Chebyshev order; ``method='exact'`` uses the full Fourier basis:
    ``||g(L) e_j||^2 = sum_n U[j, n]^2 g(e_n)^2``.  A squared norm that rounds below zero
    gives 0.
    """
    kwargs.pop("i", None)
    sq = _square_norms(g.G, g._kernels, **kwargs).cpu().numpy()
    return np.sqrt(np.maximum(sq, 0.0)).T.reshape(-1)


def compute_spectrogram(G, atom=None, M=100, **kwargs):
    r"""Squared frame norms of ``atom`` shifted along [0, lmax] (features.py:62-94).

    Column m is ``||g_m(L) e_i||^2`` with ``g_m(x) = atom(x - m lmax / (M - 1))``; the default
    atom is ``exp(-M (x / lmax)^2)``.  Returns an (N, M) float64 ndarray, also stored as
    ``G.spectr``.  ``order`` and ``method`` as in :func:`compute_norm_tig`.  All M atoms share
    one moment recurrence.  A value that rounds below zero gives 0.
    """
    lmax = G.lmax
    if not atom:
        def atom(x):
            return np.exp(-M * (x / lmax) ** 2)
    scale = np.linspace(0, lmax, M)
    kernels = [(lambda x, s=s: atom(x - s)) for s in scale]
    spectr = np.maximum(_square_norms(G, kernels, **kwargs).cpu().numpy(), 0.0)
    G.spectr = spectr
    return spectr
