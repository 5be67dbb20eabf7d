"""``pygsp/optimization.py`` on the CUDA engine: the proximal operator of graph total variation.

The reference's ``prox_tv`` (optimization.py:24-103) hands the problem to pyunlocbox's
``norm_l1`` prox and cannot run: without pyunlocbox it raises ``ImportError`` (:100), with it
``NameError`` on ``verbose`` (:102); it also reads ``G.Diff`` and an undefined ``D`` (:87, :90)
and returns nothing.  Here the problem its docstring states is solved on the device by FISTA on
the dual (csrc/tv.cu, ``gsp_prox_tv_*``), and the solution is returned.
"""
import numpy as np

from . import _native as nat
from . import utils

logger = utils.build_logger(__name__)

# iterations enqueued between two reads of the stop record
TV_BATCH = 16
_CRITS = {1: "RTOL", 2: "MAXIT"}

# the last prox_tv run: {'niter', 'crit', 'objective', 'gap'}
last_solve = None


def _apply(op, name, v, shape, dtype):
    out = op(v)
    torch = nat.require_cuda()
    if not (torch.is_tensor(out) and out.is_cuda and tuple(out.shape) == shape
            and out.dtype == dtype):
        raise TypeError("%s must map an %s CUDA tensor of %s to another one, got %r"
                        % (name, shape, dtype, type(out) if not torch.is_tensor(out) else
                           (tuple(out.shape), out.dtype, out.device)))
    return out.contiguous()


def prox_tv(x, gamma, G, A=None, At=None, nu=1, tol=10e-4, maxit=200, use_matrix=True):
    r"""Total variation proximal operator for graphs (optimization.py:24-103).

    Solves ``argmin_z 1/2 ||x - z||_2^2 + gamma ||D^T A z||_1`` with ``D^T`` the graph gradient
    (:meth:`Graph.grad`) and ``A`` an optional linear forward operator, and returns z.

    ``x``: (N,) or (N, Nsig) signal, NumPy or a CUDA tensor, not modified; the columns are
    independent problems that share one stop test on their summed objective.  Returns z of
    x's shape in the graph's dtype: NumPy in -> NumPy out, CUDA tensor in -> CUDA tensor out.

    ``A`` / ``At``: both None (identity) or both callables, each mapping an (N, Nsig) CUDA tensor
    in the graph's dtype to another one; they must be linear and adjoint to each other.  Unlike
    the reference, they receive and return CUDA tensors, not NumPy arrays.  ``nu`` bounds
    ``||A||_2^2`` (``A = s I`` takes ``nu = s**2``).  ``use_matrix`` is accepted and ignored: D
    is always a matrix in device memory.

    The method is FISTA on the dual (Beck and Teboulle's fast gradient projection), with
    K = D^T A, u in [-1, 1]^(Ne x Nsig), ``nu_bar = 2 G.lmax nu`` (the reference's ``l1_nu``,
    :82) and step ``tau = 1 / (gamma nu_bar)``::

        u_0 = u_{-1} = 0, t_0 = 1
        for k = 0, 1, ...:
            z_k   = x - gamma K* u_k
            g_k   = K z_k
            P_k   = 1/2 ||x - z_k||^2 + gamma ||g_k||_1       (summed over the columns)
            gap_k = gamma sum(|g_k| - u_k g_k)                 (>= 0 termwise)
            k >= 1: 'RTOL' if |P_k - P_{k-1}| < tol |P_k|, or P_k = P_{k-1} = 0 and tol > 0;
                    'MAXIT' if k >= maxit (checked second)  ->  return z_k, niter = k
            t_{k+1} = (1 + sqrt(1 + 4 t_k^2)) / 2,  b = (t_k - 1) / t_{k+1}
            u_{k+1} = clip(u_k + b (u_k - u_{k-1}) + tau ((1 + b) g_k - b g_{k-1}), -1, 1)

    The stop rule is the one the reference's docstring states (:53-57).  ``gap_k`` is P(z_k)
    minus the dual objective ``1/2 ||x||^2 - 1/2 ||z_k||^2``; as P is 1-strongly convex,
    ``||z_k - z*||_2 <= sqrt(2 gap_k)`` bounds the distance to the exact prox.
    ``optimization.last_solve`` then holds ``niter``, ``crit`` and the histories ``objective``
    (P_0 .. P_niter) and ``gap``.  ``gamma = 0``, ``maxit = 0`` and a graph without an edge
    between two distinct vertices return a copy of x with ``niter = 0``.

    D is computed if the graph has none (without :attr:`Graph.D`'s warning); ``G.lmax`` is
    estimated, with its warning, if it is not known.
    """
    global last_solve
    torch = nat.require_cuda()
    if (A is None) != (At is None):
        raise ValueError("A and At must both be given or both be None")
    if gamma < 0:
        raise ValueError("gamma must be non-negative, got {}".format(gamma))
    if nu <= 0:
        raise ValueError("nu must be positive, got {}".format(nu))
    if tol < 0:
        raise ValueError("tol must be non-negative, got {}".format(tol))
    if maxit < 0 or int(maxit) != maxit:
        raise ValueError("maxit must be a non-negative integer, got {}".format(maxit))
    maxit = int(maxit)
    logger.debug("use_matrix=%s is ignored: D is a matrix on the device", use_matrix)
    is_tensor = torch.is_tensor(x)
    x = G._check_signal(x)
    xt = (x if is_tensor else torch.as_tensor(np.asarray(x, dtype=np.float64))).to(
        device=G.device, dtype=G.dtype)
    one_d = xt.dim() == 1
    X = xt.reshape(G.N, -1).contiguous()
    if not bool(torch.isfinite(X).all()):
        raise ValueError("x must be finite")
    n, nsig = X.shape

    if G._D is None:
        G.compute_differential_operator()
    D = G._D
    if gamma == 0 or maxit == 0 or D.nnz == 0:
        Z = X.clone()
        last_solve = {"niter": 0, "crit": None, "objective": np.zeros(0), "gap": np.zeros(0)}
        logger.info("prox_tv: x returned unchanged (gamma = %g, maxit = %d, %d incidences)",
                    gamma, maxit, D.nnz)
    else:
        Z, rec = _solve(G, D, X, float(gamma), A, At, float(nu), float(tol), maxit)
        last_solve = rec
        logger.info("Solution found after %d iterations: objective = %e, duality gap = %e, "
                    "stopping criterion: %s", rec["niter"], rec["objective"][-1], rec["gap"][-1],
                    rec["crit"])
    out = Z[:, 0] if one_d else Z.reshape(xt.shape)
    if is_tensor:
        return out
    return out.cpu().numpy()


def _solve(G, D, X, gamma, A, At, nu, tol, maxit):
    torch = nat.require_cuda()
    n, nsig = X.shape
    ne = D.shape[1]
    Dt = D.T
    tau = 1.0 / (gamma * 2.0 * G.lmax * nu)
    sfx = nat.suffix(G.dtype)
    stream = nat.stream_ptr(G.device)
    ur = max(n, ne)
    Z = torch.empty_like(X)
    with torch.cuda.device(G.device):
        # zero state: u_0 = u_{-1} = 0, g_{-1} = 0 and the stop record; the dual blocks'
        # rows past Ne stay zero (the vertex pass reads them times 0)
        U2 = torch.zeros(2 * ur * nsig, dtype=G.dtype, device=G.device)
        Gk = torch.zeros(ne * nsig, dtype=G.dtype, device=G.device)
        blk = ur * nsig

        def u_block(k):
            return U2[(k % 2) * blk:(k % 2 + 1) * blk]

        def primal(k):
            if A is None:
                nat.call("gsp_prox_tv_primal_" + sfx, nat.i64(n), nat.i64(D.nnz), D.indptr,
                         D.indices, D.data, X, nat.i64(nsig), nat.f64(gamma), u_block(k), Z,
                         stream)
            else:
                Du = D.dot(u_block(k)[:ne * nsig].reshape(ne, nsig))
                V = _apply(At, "At", Du, (n, nsig), G.dtype)
                torch.add(X, V, alpha=-gamma, out=Z)

        def enqueue(it0, it1, cap, scal):
            if A is None:
                nat.call("gsp_prox_tv_" + sfx, nat.i64(n), nat.i64(ne), nat.i64(D.nnz), D.indptr,
                         D.indices, D.data, Dt.indptr, Dt.indices, Dt.data, X, nat.i64(nsig),
                         nat.f64(gamma), nat.f64(tau), nat.f64(tol), nat.i32(maxit), Z, U2, Gk,
                         nat.i32(it0), nat.i32(it1), nat.i32(cap), scal, stream)
            else:
                for k in range(it0, it1):
                    primal(k)
                    W = _apply(A, "A", Z, (n, nsig), G.dtype)
                    nat.call("gsp_prox_tv_edges_" + sfx, nat.i64(n), nat.i64(ne), Dt.indptr,
                             Dt.indices, Dt.data, W, X, Z, nat.i64(nsig), nat.f64(gamma),
                             nat.f64(tau), nat.f64(tol), nat.i32(maxit), U2, Gk, nat.i32(k),
                             nat.i32(cap), scal, stream)

        scal, niter, code, _ = nat.run_fista(enqueue, TV_BATCH, maxit, 2, G.device, "TV")
        crit = _CRITS[code]
        primal(niter)                    # z_niter: later vertex passes overwrote it
    hist = scal[nat.FISTA_HISTORY:nat.FISTA_HISTORY + 2 * (niter + 1)].cpu().numpy().reshape(-1, 2)
    return Z, {"niter": niter, "crit": crit, "objective": hist[:, 0].copy(),
               "gap": hist[:, 1].copy()}
