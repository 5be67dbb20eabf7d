"""``Filter``: a bank of spectral kernels applied by Chebyshev recurrence on the GPU.

Mirror of the hot-path part of ``pygsp/filters/filter.py``: the container
(:56-69), ``evaluate`` (:112-144), ``filter`` with its shape conventions
(:146-328), ``analyze`` / ``synthesize`` (:330-348), ``localize`` (:350-391)
and the small operators (:83-103).  ``method='exact'`` filters through the
Fourier basis (graphs/fourier.py) with the block kernels of csrc/block.cu.
"""
import numpy as np

from .. import _native as nat
from .. import utils
from ..graphs.graph import Graph
from . import approximations

_logger = utils.build_logger(__name__)


class Filter:
    r"""Filter bank defined by kernel functions of the graph frequencies.

    Parameters
    ----------
    G : Graph
    kernels : function or list of functions (one per filter, NumPy array in -> out)
    """

    def __init__(self, G, kernels):
        self.G = G
        single = callable(kernels) and not hasattr(kernels, "__iter__")
        self._kernels = [kernels] if single else kernels
        n_out = len(self._kernels)
        # one input feature, one output feature per kernel (an "analysis" bank)
        self.n_features_in = 1
        self.n_features_out = n_out
        self.shape = (n_out, 1)
        self.Nf = self.n_filters = n_out
        # synthesis as ONE backward recurrence (K SpMMs) instead of the reference's Nf
        # forward recurrences (Nf * K SpMMs); same value, different rounding.  Set to
        # False to reproduce the reference's operation order.
        self.fused_synthesis = True
        # a single filter is evaluated by Clenshaw's backward recurrence: 4 instead of 5
        # passes over the signal block per order (no accumulator block), same value,
        # different rounding.  False = the reference's forward recurrence and operation order.
        self.clenshaw = True

    def _get_extra_repr(self):
        return dict()

    def __repr__(self):
        fields = [("in", self.n_features_in), ("out", self.n_features_out)]
        fields += list(self._get_extra_repr().items())
        return "{}({})".format(type(self).__name__, ", ".join("%s=%s" % kv for kv in fields))

    def __len__(self):
        return self.n_filters

    def __getitem__(self, key):
        return Filter(self.G, self._kernels[key])

    def __add__(self, other):
        if not isinstance(other, Filter):
            return NotImplemented
        return Filter(self.G, self._kernels + other._kernels)

    def __call__(self, x):
        if isinstance(x, Graph):
            return Filter(x, self._kernels)
        return self.evaluate(x)

    def __matmul__(self, other):
        return self.filter(other)

    def evaluate(self, x):
        r"""Frequency response of every kernel at ``x``: shape (Nf, *x.shape)."""
        freqs = np.asanyarray(x)
        response = np.empty((self.Nf,) + freqs.shape)
        for row, g in zip(response, self._kernels):
            row[...] = g(freqs)
        return response

    def filter(self, s, method="chebyshev", order=30):
        r"""Filter signals (analysis or synthesis) -- filter.py:146-328.

        ``s`` is read as (N, N_SIGNALS, N_FEATURES).  A last dimension that is
        neither 1 nor Nf is a signal dimension.  One input feature -> analysis:
        every filter is applied, output (N, N_SIGNALS, Nf).  Nf input features
        -> synthesis: filter i is applied to feature i and the results are
        summed, output (N, N_SIGNALS).  Singleton dimensions are squeezed.
        NumPy in -> NumPy out; CUDA tensors stay on the device.
        """
        torch = nat.require_cuda()
        s = self.G._check_signal(s)
        if method not in ("chebyshev", "exact"):
            raise ValueError("Unknown method {}.".format(method))

        if s.ndim == 1 or s.shape[-1] not in [1, self.Nf]:
            if s.ndim == 3:
                raise ValueError("Third dimension (#features) should be either 1 or the number "
                                 "of filters Nf = {}, got {}.".format(self.Nf, tuple(s.shape)))
            s = s[..., None]
        n_features_in = s.shape[-1]
        if s.ndim < 3:
            s = s[:, None, :]
        if s.ndim > 3:
            raise ValueError("At most 3 dimensions: #nodes x #signals x #features.")
        n_signals = s.shape[1]
        N = self.G.N
        if method == "exact":
            return self._filter_exact(s, n_signals, n_features_in)

        c = approximations.compute_cheby_coeff(self, m=order)
        c = np.atleast_2d(np.asarray(c, dtype=np.float64))
        if c.shape[1] < 2:
            raise TypeError("The coefficients have an invalid shape")
        L = approximations._laplacian_on_device(self.G)
        view = approximations._GraphView(L)

        if n_features_in == 1:                                   # analysis
            flat = s.reshape(N, n_signals)
            if approximations._is_pinned_block(flat, L):
                # page-locked host block: column chunks, transfers overlapped with the recurrence
                from . import pipeline
                r = pipeline.filter_pinned(L, self.G.lmax, c, flat, clenshaw=self.clenshaw)
                return r.permute(1, 2, 0).squeeze()
            x, _, kind = approximations._as_device_block(view, flat)
            if self.clenshaw and c.shape[0] == 1:
                r = approximations.cheby_clenshaw_device(L, self.G.lmax, c, x)[None]
            elif c.shape[0] > approximations.WIDE_BANK:
                r = approximations.cheby_bank_device(L, self.G.lmax, c, x)
            else:
                r = approximations.cheby_op_device(L, self.G.lmax, c, x)  # (Nf, N, nsig)
            out = r.permute(1, 2, 0)                                      # (N, nsig, Nf)
        else:                                                    # synthesis
            x, _, kind = approximations._as_device_block(view, s.reshape(N, -1))
            x = x.reshape(N, n_signals, n_features_in)
            if self.fused_synthesis and n_features_in <= approximations.WIDE_BANK:
                out = approximations.cheby_clenshaw_device(L, self.G.lmax, c, x.permute(2, 0, 1))
            elif self.fused_synthesis:
                out = approximations.cheby_synthesis_wide_device(L, self.G.lmax, c,
                                                                 x.permute(2, 0, 1))
            else:
                out = torch.zeros((N, n_signals), dtype=L.dtype, device=L.device)
                for i in range(n_features_in):
                    xi = x[:, :, i].contiguous()
                    out += approximations.cheby_op_device(L, self.G.lmax, c[i], xi)[0]
            out = out[:, :, None]
        out = out.squeeze()
        return approximations._leave_device(out, kind)

    def _filter_exact(self, s, n_signals, n_features_in):
        """filter.py:292-301: s_hat = U^T s, times the responses at G.e, back by U."""
        from ..graphs import fourier
        torch = nat.require_cuda()
        G, N = self.G, self.G.N
        n_features_out = self.Nf if n_features_in == 1 else 1
        f = self.evaluate(G.e)                                    # (Nf, len(e))
        assert f.T.shape == (N, self.Nf), "method='exact' needs the full Fourier basis"
        U = G._device_basis()
        x, _, kind = approximations._as_device_block(
            approximations._GraphView(G.L), s.reshape(N, n_signals * n_features_in))
        s_hat = fourier.block_gram(U, x).reshape(N, n_signals, n_features_in)
        f = torch.from_numpy(np.ascontiguousarray(f.T)).to(s_hat.device)   # (N, Nf) float64
        if n_features_in == 1:                                   # analysis
            out_hat = s_hat * f[:, None, :]
        else:                                                    # synthesis
            out_hat = (s_hat * f[:, None, :]).sum(dim=2, keepdim=True)
        out = fourier.block_combine(U, out_hat.reshape(N, n_signals * n_features_out))
        out = out.reshape(N, n_signals, n_features_out).squeeze()
        return approximations._leave_device(out, kind)

    def analyze(self, s, method="chebyshev", order=30):
        r"""Alias of :meth:`filter` for single-feature input (filter.py:330-336)."""
        if s.ndim == 3 and s.shape[-1] != 1:
            raise ValueError("Last dimension (#features) should be 1, got {}.".format(
                tuple(s.shape)))
        return self.filter(s, method, order)

    def synthesize(self, s, method="chebyshev", order=30):
        r"""Alias of :meth:`filter` for Nf-feature input (filter.py:338-348)."""
        if s.shape[-1] != self.Nf:
            raise ValueError("Last dimension (#features) should be the number of filters "
                             "Nf = {}, got {}.".format(self.Nf, tuple(s.shape)))
        return self.filter(s, method, order)

    def compute_frame(self, **kwargs):
        r"""Matrix of the analysis operator, (N Nf, N): one delta per vertex through
        :meth:`filter` (filter.py:540-603)."""
        if self.G.N > 2000:
            _logger.warning("Creating a big matrix. You should prefer the filter method.")
        s = np.identity(self.G.N)
        return self.filter(s, **kwargs).T.reshape(-1, self.G.N)

    def toarray(self):
        r"""Array representation of the bank: :meth:`compute_frame` (filter.py:105-110)."""
        return self.compute_frame()

    def localize(self, i, **kwargs):
        r"""Kernels localised at vertex ``i``: sqrt(N) g(L) delta_i (filter.py:350-391)."""
        delta = np.zeros(self.G.N)
        delta[i] = 1
        return self.filter(delta, **kwargs) * np.sqrt(self.G.N)

    # ------------------------------------------------------------------------ frames
    def estimate_frame_bounds(self, x=None):
        r"""Frame bounds (A, B): the extrema over ``x`` of ``sum_i g_i(x)^2`` (filter.py:393-504).

        ``x`` defaults to 1000 evenly spaced points of [0, lmax]; pass ``G.e`` for the exact
        bounds on the graph's spectrum.  Host NumPy on the responses.
        """
        x = np.linspace(0, self.G.lmax, 1000) if x is None else np.asanyarray(x)
        energy = np.sum(self.evaluate(x) ** 2, axis=0)
        return energy.min(), energy.max()

    def complement(self, frame_bound=None):
        r"""The filter that makes the bank a tight frame: ``sqrt(B - sum_i g_i(x)^2)``
        (filter.py:602-661).

        ``B`` is ``frame_bound``, or the largest energy among the frequencies the complement is
        evaluated at when it is None.  A bound below that energy raises ``ValueError`` when the
        complement is evaluated.
        """
        def kernel(x):
            energy = np.sum(self.evaluate(x) ** 2, axis=0)
            peak = energy.max()
            if frame_bound is None:
                bound = peak
            elif peak > frame_bound:
                raise ValueError("The chosen bound is not feasible. "
                                 "Choose at least {}.".format(peak))
            else:
                bound = frame_bound
            return np.sqrt(bound - energy)

        return Filter(self.G, kernel)

    def inverse(self):
        r"""The bank whose synthesis inverts this bank's analysis (filter.py:663-759).

        At every frequency the responses h(x) of the inverse are the pseudo-inverse of the column
        g(x) of this bank's responses: ``h_i(x) = g_i(x) / sum_j g_j(x)^2``, and 0 where every
        g_j(x) is 0.  A warning is logged when the frame bounds (on [0, lmax]) say the bank is not
        a frame (A = 0) or is badly conditioned (A / B < 1e-10).
        """
        A, B = self.estimate_frame_bounds()
        if A == 0:
            _logger.warning("The filter bank is not invertible as it is not "
                            "a frame (lower frame bound A=0).")
        elif A / B < 1e-10:
            _logger.warning("The filter bank is badly conditioned. "
                            "The inverse will be approximate.")

        def kernel(x, i):
            g = self.evaluate(x)
            energy = np.sum(g ** 2, axis=0)
            safe = np.where(energy > 0, energy, 1.0)
            return np.where(energy > 0, g[i] / safe, 0.0)

        return Filter(self.G, [lambda x, i=i: kernel(x, i) for i in range(self.n_filters)])
