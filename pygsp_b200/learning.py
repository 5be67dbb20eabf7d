"""``pygsp/learning.py`` on the CUDA engine: Tikhonov regression / classification on graphs.

``regression_tikhonov`` (learning.py:255-365) minimises ``|Mx - y|^2 + tau x'Lx``.  The
reference solves ``(M + tau L) x = M y`` with ``scipy.sparse.linalg.cg``, one column at a
time in a Python loop, every product a SciPy SpMV (learning.py:326-337); for ``tau = 0`` it
solves the harmonic extension ``L_uu x_u = -L_ul y_l`` with a sparse direct solver (:350-365).
Here both are ONE block conjugate-gradient run on the device (``gsp_cg_*``, csrc/cg.cu): all
columns advance together, the product with L is the SpMM step kernel of the filter path.

``classification_tikhonov_simplex`` (learning.py:42-180) hands its problem to pyunlocbox's
accelerated forward-backward solver; here that solver runs on the device (``gsp_fb_simplex_*``,
csrc/simplex.cu) with its stopping rules, and pyunlocbox is not needed.
"""
import numpy as np

from . import _native as nat
from . import utils

logger = utils.build_logger(__name__)

# iterations enqueued between two reads of the simplex solver's stop record
SIMPLEX_BATCH = 16
MAX_CLASSES = 256
_CRITS = {1: "ATOL", 2: "DTOL", 3: "RTOL", 4: "XTOL", 5: "MAXIT"}
_SOLVE_DEFAULTS = {"atol": None, "dtol": None, "rtol": 1e-3, "xtol": None, "maxit": 200,
                   "verbosity": "LOW"}

# the last classification_tikhonov_simplex run: {'niter', 'crit', 'objective', 'batches'}
last_solve = None


def _to_logits(x):
    logits = np.zeros([len(x), np.max(x) + 1])
    logits[range(len(x)), x] = 1
    return logits


def classification_tikhonov(G, y, M, tau=0):
    r"""Classification by Tikhonov regression on the one-hot logits (learning.py:176-252)."""
    y = np.array(y, copy=True)
    y[np.asarray(M) == False] = 0  # noqa: E712
    Y = _to_logits(y.astype(int))
    return regression_tikhonov(G, Y, M, tau)


def classification_tikhonov_simplex(G, y, M, tau=0.1, **kwargs):
    r"""Classification with class probabilities by Tikhonov minimisation (learning.py:42-180).

    ``argmin_X ||M X - Y||^2 + tau tr(X'LX)`` with every row of X on the probability simplex
    (``X >= 0``, rows summing to 1), Y the one-hot logits of the labels ``y`` (C = max label + 1
    classes, at most 256).  Solved by accelerated forward-backward (FISTA) from ``X = Y`` with
    step ``0.5 / (1 + tau G.lmax)``, as the reference does with pyunlocbox.  ``y``: (N,)
    measurements (entries where ``M`` is False are ignored and may be NaN), ``M``: boolean mask
    of length N; the inputs are not modified.  Keywords are pyunlocbox's ``solve`` stopping
    parameters: ``atol``, ``dtol``, ``rtol`` (default 1e-3), ``xtol``, ``maxit`` (default 200)
    and ``verbosity`` ('NONE', 'LOW', 'HIGH', 'ALL': what is logged).  Returns the (N, C) X;
    NumPy in -> NumPy out (float64 for a float64 graph, else float32), CUDA tensor in -> CUDA
    tensor out.  ``learning.last_solve`` then holds the iteration count, the stopping criterion
    and the objective at every iterate.
    """
    global last_solve
    unknown = sorted(set(kwargs) - set(_SOLVE_DEFAULTS))
    if unknown:
        raise TypeError("classification_tikhonov_simplex() got an unexpected keyword argument "
                        "'%s'" % unknown[0])
    if tau <= 0:
        raise ValueError("Tau should be greater than 0.")
    opts = dict(_SOLVE_DEFAULTS, **kwargs)
    if opts["verbosity"] not in ("NONE", "LOW", "HIGH", "ALL"):
        raise ValueError("Verbosity should be either NONE, LOW, HIGH or ALL.")
    if all(opts[k] is None for k in ("atol", "dtol", "rtol", "xtol", "maxit")):
        raise ValueError("at least one stopping criterion (atol, dtol, rtol, xtol, maxit) is needed")
    torch = nat.require_cuda()
    is_tensor = torch.is_tensor(y)
    M_host = np.asarray(M.cpu() if torch.is_tensor(M) else M)
    if M_host.size != G.n_vertices:
        raise ValueError("M should be of size [G.n_vertices,]")
    mask = torch.as_tensor(M_host.astype(bool).ravel(), device=G.device)
    yt = (y if is_tensor else torch.as_tensor(np.asarray(y, dtype=np.float64))).to(
        device=G.device, dtype=torch.float64).reshape(-1)
    if yt.numel() != G.n_vertices:
        raise ValueError("y should be of size [G.n_vertices,]")
    yt = torch.where(mask, yt, torch.zeros_like(yt))         # learning.py:117 (NaNs dropped)
    if bool(torch.isnan(yt).any()):
        raise ValueError("labelled vertices must have a label (got NaN)")
    lab = yt.to(torch.int64)                                 # y.astype(int): toward zero
    if bool((lab < 0).any()):
        raise ValueError("labels must be non-negative integers")
    C = int(lab.max()) + 1
    if C > MAX_CLASSES:
        raise ValueError("at most %d classes are supported, got %d" % (MAX_CLASSES, C))
    label = torch.where(mask, lab, torch.full_like(lab, -1)).to(torch.int32).contiguous()

    step = 0.5 / (1 + tau * G.lmax)
    n, L = G.n_vertices, G.L
    maxit = opts["maxit"]
    # iteration k's objective is formed by the k-th row pass: maxit stops by pass max(maxit, 1)
    last_pass = None if maxit is None else max(int(maxit), 1)
    tol = np.array([np.nan if opts[k] is None else float(opts[k])
                    for k in ("atol", "dtol", "rtol", "xtol")], dtype=np.float64)
    X2 = torch.empty(2 * n * C, dtype=G.dtype, device=G.device)
    LX2 = torch.empty_like(X2)
    plan = L.tile_plan(C, 0)

    def enqueue(it0, it1, cap, scal):
        nat.call("gsp_fb_simplex_" + nat.suffix(G.dtype), nat.i64(n), nat.i64(L.nnz), L.indptr,
                 L.indices, L.data, label, nat.i64(C), nat.f64(tau), nat.f64(step), tol,
                 nat.i32(-1 if maxit is None else maxit), X2, LX2, nat.i32(it0), nat.i32(it1),
                 nat.i32(cap), scal, plan, nat.stream_ptr(G.device))

    with torch.cuda.device(G.device):
        scal, niter, code, batches = nat.run_fista(enqueue, SIMPLEX_BATCH, last_pass, 1, G.device,
                                                   "simplex")
    crit = _CRITS[code]
    obj = scal[nat.FISTA_HISTORY:nat.FISTA_HISTORY + niter + 1].cpu().numpy()
    last_solve = {"niter": niter, "crit": crit, "objective": obj, "batches": batches}
    if opts["verbosity"] in ("HIGH", "ALL"):
        for k in range(1, niter + 1):
            logger.info("iteration %d: objective = %.2e", k, obj[k])
    if opts["verbosity"] != "NONE":
        logger.info("Solution found after %d iterations: objective f(sol) = %e, stopping "
                    "criterion: %s", niter, obj[-1], crit)
    X = X2[(niter % 2) * n * C:(niter % 2 + 1) * n * C].reshape(n, C).clone()
    if is_tensor:
        return X
    return X.cpu().numpy().astype(np.float64 if G.dtype == torch.float64 else np.float32)


def _block_cg(G, tau, row_scale, diag, B, tol, maxiter, patience=8):
    """Solve (diag(row_scale) tau L + diag(diag)) X = B on the device; B (N, nsig) tensor.
    Stops early when the worst residual has not halved over ``patience`` batches of 25
    iterations."""
    torch = nat.require_cuda()
    L = G.L
    n, nsig = B.shape
    cap = int(maxiter)
    X = torch.empty_like(B)
    R, P, Q = torch.empty_like(B), torch.empty_like(B), torch.empty_like(B)
    scal = torch.zeros((cap + 1 + 2048) * nsig, dtype=torch.float64, device=B.device)
    done, batch = 0, 25
    best, stall = None, 0
    while done < cap:
        nxt = min(cap, done + batch)
        with torch.cuda.device(B.device):
            nat.call("gsp_cg_" + nat.suffix(B.dtype), nat.i64(n), nat.i64(L.nnz), L.indptr, L.indices,
                     L.data, nat.f64(tau), row_scale, diag, B, X, R, P, Q, nat.i64(nsig),
                     nat.i32(done), nat.i32(nxt), nat.i32(cap), scal, nat.stream_ptr(B.device))
        done = nxt
        rr = scal[:(done + 1) * nsig].reshape(done + 1, nsig).cpu().numpy()
        rel = np.sqrt(rr[-1] / np.maximum(rr[0], 1e-300))
        worst = float(rel.max())
        if worst <= tol:
            return X, done, worst
        if best is None or worst < 0.5 * best:             # float32 stagnates above tiny tols
            best, stall = worst, 0
        else:
            stall += 1
            if stall >= patience:
                break
    logger.warning("conjugate gradients stopped at relative residual %.2e after %d iterations",
                   worst, done)
    return X, done, worst


def regression_tikhonov(G, y, M, tau=0, *, tol=None, maxiter=None):
    r"""Solve a regression problem on a graph via Tikhonov minimisation (learning.py:255-365).

    ``argmin_x |Mx - y|^2 + tau x'Lx`` for ``tau > 0``;
    ``argmin_x x'Lx  s.t.  y = Mx`` otherwise.  ``y``: (N,) or (N, Nv) measurements (entries where
    ``M`` is False are ignored and may be NaN), ``M``: boolean mask of length N.  The inputs are
    not modified.  ``tol``: relative residual at which CG stops (default 1e-6 for a float32
    graph, 1e-10 for float64; the reference's SciPy default is 1e-5).  NumPy in -> NumPy out,
    CUDA tensor in -> CUDA tensor out.
    """
    torch = nat.require_cuda()
    is_tensor = torch.is_tensor(y)
    M_host = np.asarray(M.cpu() if torch.is_tensor(M) else M)
    if M_host.size != G.n_vertices:
        raise ValueError("M should be of size [G.n_vertices,]")
    mask = torch.as_tensor(M_host.astype(bool).ravel(), device=G.device)
    yt = (y if is_tensor else torch.as_tensor(np.asarray(y, dtype=np.float64))).to(
        device=G.device, dtype=G.dtype)
    one_d = yt.dim() == 1
    Y = yt.reshape(G.N, -1).clone()
    Y[~mask] = 0                                            # learning.py:321-322 / :358 (NaNs dropped)
    if tol is None:
        tol = 1e-6 if G.dtype == torch.float32 else 1e-10
    if maxiter is None:
        maxiter = int(min(10 * G.N, 4000))                 # SciPy's default is 10 N
    m = mask.to(G.dtype)
    out = torch.empty_like(Y)
    for lo in range(0, Y.shape[1], 256):                    # block CG: <= 256 columns at a time
        B = Y[:, lo:lo + 256].contiguous()
        if tau > 0:
            X, _, _ = _block_cg(G, float(tau), None, m, B, tol, maxiter)
            out[:, lo:lo + 256] = X
        else:
            # harmonic extension: CG on L restricted to the unlabelled vertices, written on
            # full-length vectors (identity on the labelled ones)
            rhs = -(G.L.dot(B)) * (1 - m)[:, None]
            X, _, _ = _block_cg(G, 1.0, (1 - m).contiguous(), m, rhs.contiguous(), tol, maxiter)
            out[:, lo:lo + 256] = B + X * (1 - m)[:, None]
    if one_d:
        out = out[:, 0]
    if is_tensor:
        return out
    return out.cpu().numpy().astype(np.float64 if G.dtype == torch.float64 else np.float32)
