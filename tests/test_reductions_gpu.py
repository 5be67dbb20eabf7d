"""The fixed-order column reductions of csrc/reduce.cuh and the kernels built on them, called
directly: block_gram / block_combine / block_residual (csrc/block.cu), the Chebyshev moments
pass (csrc/moments.cu), the Krylov combine (csrc/krylov.cu), the block CG (csrc/cg.cu) and the
FISTA last-block reduction of simplex classification and prox_tv.

Two kinds of reference, so that a failure always means the kernel is wrong:

* exact arithmetic: small integer entries, so every product and partial sum is an integer far
  below 2^53 (2^24 for float32 outputs) and the exact answer is the same in any order;
* restated order: float32-valued data, whose pairwise products are exact in float64, so only the
  order of the additions is left, and oracle/reduce_oracle.py restates it.

The row counts put n at every edge of the partition (1 .. 264 parts, the 8-wide loop of sum_parts
with and without its tail, chunks below, at and above 1024 rows and of every residue mod 32), the
widths at every column group, micro tile and slab edge."""
import ctypes

import numpy as np
import pytest
from scipy import sparse
from scipy.sparse import linalg as sla

from oracle import learning_oracle as lo
from oracle import optimization_oracle as oo
from oracle import difference_oracle as do
from oracle import reduce_oracle as ro

pytestmark = pytest.mark.gpu

F64, F32 = np.float64, np.float32

WIDTHS = (1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 257)
SLAB_WIDTHS = (15, 16, 17, 31, 32, 33)
BLOCK_ROWS = (1, 15, 16, 17, 31, 32, 33, 127, 128, 129, 8 * 32 - 1, 8 * 32 + 1, 70001, 10**6)
PARTITION_ROWS = (1, 7, 8, 9, 1023, 1024, 1025, 2049, 7 * 1024, 8 * 1024 - 1, 8 * 1024,
                  8 * 1024 + 1, 16 * 1024, 16 * 1024 + 5, 262 * 1024 + 1, 263 * 1024 + 1,
                  264 * 1024, 264 * 1024 + 1, 10**6 + 3)
RESIDUE_ROWS = tuple(range(1025, 1088))          # two parts; the chunk takes every residue mod 32
COLS = (1, 31, 32, 33, 65)
WIDE_ROWS_COLS = (1, 33)                         # widths at n >= 262 * 1024
EDGE_COLS = (0, 1, 30, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128)


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


@pytest.fixture(scope="module")
def nat(gsp):
    from pygsp_b200 import _native
    _native.lib().gsp_launch_count.restype = ctypes.c_uint64
    return _native


@pytest.fixture(scope="module")
def sms(nat):
    count = ctypes.c_int()
    nat.call("gsp_device_info", ctypes.byref(count), None, None, None)
    return count.value


def tdtype(dt):
    import torch
    return torch.float64 if dt == F64 else torch.float32


def dev(a, dt):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a), device="cuda").to(tdtype(dt))


def host(t):
    return t.cpu().numpy().astype(np.float64)


def bits(a):
    return np.ascontiguousarray(np.asarray(a, dtype=np.float64)).view(np.uint64)


def assert_bits(got, ref):
    got, ref = np.asarray(got, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape
    bad = bits(got) != bits(ref)
    assert not bad.any(), (np.argwhere(bad)[:5], got[bad][:5], ref[bad][:5])


def cols_for(n):
    return WIDE_ROWS_COLS if n >= 262 * 1024 else COLS


# ------------------------------------------------------------------ block_gram, block_combine
@pytest.mark.parametrize("dt", [F64, F32])
def test_gram_and_combine_every_width_pair(gsp, dt):
    """Every micro tile (2, 4, 8), multi-tile grids and the combine's slab tails, exactly."""
    from pygsp_b200.graphs import fourier as fr
    rng = np.random.default_rng(1)
    n = 300
    A = rng.integers(-4, 5, size=(n, 257)).astype(F64)
    B = rng.integers(-4, 5, size=(n, 257)).astype(F64)
    Q = rng.integers(-4, 5, size=(257, 257)).astype(F64)
    Ad = {ka: dev(A[:, :ka], dt) for ka in set(WIDTHS) | set(SLAB_WIDTHS)}
    Bd = {kb: dev(B[:, :kb], dt) for kb in WIDTHS}
    for ka in WIDTHS:
        for kb in WIDTHS:
            C = fr.block_gram(Ad[ka], Bd[kb])
            assert_bits(host(C), A[:, :ka].T @ B[:, :kb])
    for ka in sorted(set(WIDTHS) | set(SLAB_WIDTHS)):
        for kq in WIDTHS:
            Y = fr.block_combine(Ad[ka], Q[:ka, :kq])
            assert Y.dtype == tdtype(dt)
            assert_bits(host(Y), A[:, :ka] @ Q[:ka, :kq])


@pytest.mark.parametrize("dt", [F64, F32])
def test_gram_and_combine_every_row_count(gsp, dt):
    """Slab depths 16 / 32, row tiles 32 / 64 / 128, one Gram part and many, exactly."""
    from pygsp_b200.graphs import fourier as fr
    rng = np.random.default_rng(2)
    big = max(BLOCK_ROWS)
    A = rng.integers(-4, 5, size=(big, 129)).astype(np.int8)
    B = rng.integers(-4, 5, size=(big, 128)).astype(np.int8)
    Ad, Bd = dev(A, dt), dev(B, dt)
    for n in BLOCK_ROWS:
        shapes = ((1, 1), (33, 31), (17, 64), (64, 65), (129, 128), (3, 128))
        if n > 10**5:
            shapes = shapes[:3]
        for ka, kb in shapes:
            An, Bn = A[:n, :ka].astype(F64), B[:n, :kb].astype(F64)
            C = fr.block_gram(Ad[:n, :ka], Bd[:n, :kb])
            assert_bits(host(C), An.T @ Bn)
            Q = rng.integers(-4, 5, size=(ka, kb)).astype(F64)
            Y = fr.block_combine(Ad[:n, :ka], Q)
            assert_bits(host(Y), An @ Q)


def test_block_wrappers_refuse_mismatched_operands(gsp, nat):
    import torch
    from pygsp_b200.graphs import fourier as fr
    A32 = torch.zeros((40, 3), dtype=torch.float32, device="cuda")
    A64 = torch.zeros((40, 3), dtype=torch.float64, device="cuda")
    before = nat.lib().gsp_launch_count()
    bad = [lambda: fr.block_gram(A32, A64),
           lambda: fr.block_gram(A64, A64[:39]),
           lambda: fr.block_gram(A64, A64.cpu()),
           lambda: fr.block_combine(A64, np.zeros((4, 2))),
           lambda: fr.block_combine(A64, np.zeros((2, 2))),
           lambda: fr.block_residual(A64, A32, np.zeros(3)),
           lambda: fr.block_residual(A64, A64[:39], np.zeros(3)),
           lambda: fr.block_residual(A64, A64[:, :2], np.zeros(3)),
           lambda: fr.block_residual(A64, A64, np.zeros(2)),
           lambda: fr.block_residual(A64, A64, np.zeros(4))]
    for call in bad:
        with pytest.raises(ValueError):
            call()
    assert nat.lib().gsp_launch_count() == before


@pytest.mark.parametrize("dt", [F64, F32])
def test_block_residual_takes_strided_blocks(gsp, dt):
    rng = np.random.default_rng(3)
    from pygsp_b200.graphs import fourier as fr
    X = dev(rng.standard_normal((5000, 66)).astype(F32), dt)
    LX = dev(rng.standard_normal((5000, 66)).astype(F32), dt)
    theta = rng.standard_normal(33)
    got = fr.block_residual(X[:, ::2], LX[:, 1::2], theta)
    assert_bits(got, fr.block_residual(X[:, ::2].contiguous(), LX[:, 1::2].contiguous(), theta))


# ------------------------------------------------------------- block_residual, moments_step
@pytest.fixture(scope="module")
def partition_blocks():
    """Integer and float32-valued (n, 65) operands for the largest partition row count."""
    rng = np.random.default_rng(4)
    n = max(PARTITION_ROWS)
    return {"int": (rng.integers(-4, 5, size=(n, 65)).astype(np.int8),
                    rng.integers(-4, 5, size=(n, 65)).astype(np.int8)),
            "float": (rng.standard_normal((n, 65), dtype=np.float32),
                      rng.standard_normal((n, 65), dtype=np.float32))}


def moments(nat, tn, tc, m=1, k=0, sums=None):
    """gsp_cheby_moments_step on device blocks tn, tc: the (m, 2, b) sums array."""
    import torch
    n, b = tn.shape
    if sums is None:
        sums = torch.full((m, 2, b), float("nan"), dtype=torch.float64, device="cuda")
    nat.call("gsp_cheby_moments_step_" + nat.suffix(tn.dtype), nat.i64(n), tn.contiguous(),
             tc.contiguous(), nat.i64(b), nat.i32(m), nat.i32(k), sums, nat.stream_ptr())
    return sums


def partition_cases():
    for n in PARTITION_ROWS:
        for k in cols_for(n):
            yield n, k
    for n in RESIDUE_ROWS:
        for k in (1, 33):
            yield n, k


@pytest.mark.parametrize("kind", ["exact", "order"])
def test_block_residual_partition_edges(gsp, partition_blocks, kind):
    """Exact: integer X, LX and theta.  Restated order: theta = 0, so the term is LX^2, exact
    for float32-valued data (a nonzero theta rounds LX - theta X before the square)."""
    from pygsp_b200.graphs import fourier as fr
    Xh, LXh = partition_blocks["int" if kind == "exact" else "float"]
    theta = np.resize(np.arange(-3, 4, dtype=F64), 65) if kind == "exact" else np.zeros(65)
    for dt in (F64, F32):
        Xd, LXd = dev(Xh, dt), dev(LXh, dt)
        for n, k in partition_cases():
            got = fr.block_residual(Xd[:n, :k], LXd[:n, :k], theta[:k])
            if kind == "exact":
                d = LXh[:n, :k].astype(np.int64) - theta[:k].astype(np.int64) * Xh[:n, :k]
                ref = (d * d).sum(axis=0)
            else:
                v = LXh[:n, :k].astype(F64)
                ref = ro.column_sums(v * v)
            assert_bits(got, ref)
        del Xd, LXd


@pytest.mark.parametrize("kind", ["exact", "order"])
def test_moments_step_partition_edges(gsp, nat, partition_blocks, kind):
    """Both sums, ||t_next||^2 and <t_next, t_cur>, exactly and in the restated order."""
    Th, Ch = partition_blocks["int" if kind == "exact" else "float"]
    for dt in (F64, F32):
        Td, Cd = dev(Th, dt), dev(Ch, dt)
        for n, k in partition_cases():
            got = host(moments(nat, Td[:n, :k], Cd[:n, :k])[0])
            a, c = Th[:n, :k].astype(F64), Ch[:n, :k].astype(F64)
            if kind == "exact":
                ref = np.stack([(a * a).sum(axis=0), (a * c).sum(axis=0)])
            else:
                ref = np.stack([ro.column_sums(a * a), ro.column_sums(a * c)])
            assert_bits(got, ref)
        del Td, Cd


@pytest.mark.parametrize("dt", [F64, F32])
def test_moments_step_lands_at_step_k(gsp, nat, dt):
    import torch
    rng = np.random.default_rng(5)
    a = rng.integers(-4, 5, size=(3000, 33)).astype(F64)
    c = rng.integers(-4, 5, size=(3000, 33)).astype(F64)
    ref = np.stack([(a * a).sum(axis=0), (a * c).sum(axis=0)])
    m = 5
    sums = torch.full((m, 2, 33), float("nan"), dtype=torch.float64, device="cuda")
    for k in (3, 0, 4):
        moments(nat, dev(a, dt), dev(c, dt), m, k, sums)
    got = host(sums)
    for k in range(m):
        if k in (0, 3, 4):
            assert_bits(got[k], ref)
        else:
            assert np.isnan(got[k]).all()


@pytest.mark.parametrize("b", [1, 31, 32, 33, 64, 65, 129])
def test_columns_are_independent(gsp, nat, b):
    """A column's bits equal its bits computed alone and at the mirrored position (the header's
    guarantee, checked without restating the order)."""
    from pygsp_b200.graphs import fourier as fr
    rng = np.random.default_rng(b)
    n = 70001
    X = rng.standard_normal((n, b))
    LX = rng.standard_normal((n, b))
    theta = rng.standard_normal(b)
    for dt in (F64, F32):
        Xd, LXd = dev(X, dt), dev(LX, dt)
        res = fr.block_residual(Xd, LXd, theta)
        mom = host(moments(nat, LXd, Xd)[0])
        res_rev = fr.block_residual(Xd.flip(1), LXd.flip(1), theta[::-1])
        mom_rev = host(moments(nat, LXd.flip(1), Xd.flip(1))[0])
        for j in [j for j in EDGE_COLS if j < b] + [b - 1]:
            alone = fr.block_residual(Xd[:, j:j + 1], LXd[:, j:j + 1], theta[j:j + 1])
            assert_bits(alone, res[j:j + 1])
            assert_bits(res_rev[b - 1 - j], res[j])
            alone = host(moments(nat, LXd[:, j:j + 1], Xd[:, j:j + 1])[0])
            assert_bits(alone, mom[:, j:j + 1])
            assert_bits(mom_rev[:, b - 1 - j], mom[:, j])


@pytest.mark.parametrize("dt", [F64, F32])
def test_probe_block(gsp, nat, dt):
    import torch
    for n, v0, b in ((1, 0, 1), (5, 2, 3), (4099, 0, 33), (4099, 4066, 33), (4099, 1000, 129)):
        X = torch.full((n, b), float("nan"), dtype=tdtype(dt), device="cuda")
        nat.call("gsp_probe_block_" + nat.suffix(X.dtype), nat.i64(n), nat.i64(v0), nat.i64(b), X,
                 nat.stream_ptr())
        assert_bits(host(X), np.eye(n)[:, v0:v0 + b])


@pytest.mark.parametrize("m", [1, 2, 30])
def test_moments_finish(gsp, nat, m):
    import torch
    rng = np.random.default_rng(m)
    n, v0, b = 300, 7, 65
    sums = rng.standard_normal((m, 2, b))
    mu = torch.full((n, 2 * m + 1), float("nan"), dtype=torch.float64, device="cuda")
    nat.call("gsp_cheby_moments_finish", nat.i64(n), nat.i32(m), nat.i64(v0), nat.i64(b),
             torch.as_tensor(sums, device="cuda"), mu, nat.stream_ptr())
    ref = np.full((n, 2 * m + 1), np.nan)
    mu1 = sums[0, 1]
    ref[v0:v0 + b, 0] = 1.0
    ref[v0:v0 + b, 1] = mu1
    for k in range(1, m + 1):
        ref[v0:v0 + b, 2 * k] = 2.0 * sums[k - 1, 0] - 1.0
        if k < m:
            ref[v0:v0 + b, 2 * k + 1] = 2.0 * sums[k, 1] - mu1
    got = mu.cpu().numpy()
    assert_bits(np.nan_to_num(got, nan=7.5), np.nan_to_num(ref, nan=7.5))


# ------------------------------------------------------------------------------ Krylov combine
@pytest.mark.parametrize("dt", [F64, F32])
def test_krylov_combine(gsp, nat, dt):
    """Filter tiles of 16, column groups of 32, padding columns of Y left untouched."""
    import torch
    rng = np.random.default_rng(6)
    n = 1001
    for nf in (1, 15, 16, 17, 33):
        for ns in (1, 31, 32, 33):
            for kb in (1, 2, 30):
                V = rng.integers(-4, 5, size=(kb, n, ns)).astype(F64)
                W = rng.integers(-4, 5, size=(nf, kb, ns)).astype(F64)
                ldy = ns + 3
                Y = torch.full((nf, n, ldy), float("nan"), dtype=tdtype(dt), device="cuda")
                nat.call("gsp_krylov_combine_" + nat.suffix(Y.dtype), nat.i64(n), dev(V, dt),
                         nat.i64(kb), torch.as_tensor(W, device="cuda"), nat.i64(nf), nat.i64(ns),
                         Y, nat.i64(ldy), nat.stream_ptr())
                got = host(Y)
                assert_bits(got[:, :, :ns], np.einsum("irj,fij->frj", V, W))
                assert np.isnan(got[:, :, ns:]).all()


# -------------------------------------------------------------------------------- block CG
def banded_edges(n, seed):
    """Edges i ~ i + 1, i + 3, i + 7 of a connected banded graph, integer weights 1 or 2."""
    rng = np.random.default_rng(seed)
    r = np.concatenate([np.arange(n - s) for s in (1, 3, 7) if s < n] + [np.zeros(0, int)])
    c = np.concatenate([np.arange(s, n) for s in (1, 3, 7) if s < n] + [np.zeros(0, int)])
    return r, c, rng.integers(1, 3, r.size).astype(F64)


def banded_adjacency(n, seed):
    r, c, w = banded_edges(n, seed)
    W = sparse.coo_matrix((np.r_[w, w], (np.r_[r, c], np.r_[c, r])), shape=(n, n)).tocsr()
    W.sort_indices()
    return W


def banded_laplacian(n, seed):
    """Combinatorial Laplacian of banded_adjacency(n, seed), diagonal stored even where it is 0:
    integer entries, so L 1 = 0 exactly."""
    r, c, w = banded_edges(n, seed)
    deg = np.bincount(r, w, n) + np.bincount(c, w, n)
    idx = np.arange(n)
    L = sparse.coo_matrix((np.concatenate([deg, -w, -w]),
                           (np.concatenate([idx, r, c]), np.concatenate([idx, c, r]))),
                          shape=(n, n)).tocsr()
    L.sort_indices()
    return L


class DeviceL:
    def __init__(self, L, dt):
        import torch
        self.n, self.nnz = L.shape[0], L.nnz
        self.indptr = torch.as_tensor(L.indptr.astype(np.int32), device="cuda")
        self.indices = torch.as_tensor(L.indices.astype(np.int32), device="cuda")
        self.data = dev(L.data, dt)


class CG:
    """A block CG run of gsp_cg on device operands; run(it0, it1) enqueues [it0, it1)."""

    def __init__(self, nat, Ld, tau, a, d, B, cap):
        import torch
        self.nat, self.Ld, self.tau, self.a, self.d, self.B, self.cap = nat, Ld, tau, a, d, B, cap
        self.X, self.R, self.P, self.Q = (torch.empty_like(B) for _ in range(4))
        self.scal = torch.zeros((cap + 1 + 2048) * B.shape[1], dtype=torch.float64, device="cuda")

    def run(self, it0, it1):
        nat, Ld, (n, nsig) = self.nat, self.Ld, self.B.shape
        nat.call("gsp_cg_" + nat.suffix(self.B.dtype), nat.i64(n), nat.i64(Ld.nnz), Ld.indptr,
                 Ld.indices, Ld.data, nat.f64(self.tau), self.a, self.d, self.B, self.X, self.R,
                 self.P, self.Q, nat.i64(nsig), nat.i32(it0), nat.i32(it1), nat.i32(self.cap),
                 self.scal, nat.stream_ptr())
        return self

    def rr(self):
        """The rr history, (cap + 1, nsig)."""
        return self.scal[:(self.cap + 1) * self.B.shape[1]].reshape(self.cap + 1, -1).cpu().numpy()


def cg(nat, Ld, tau, a, d, B, ranges, cap):
    """gsp_cg over the iteration ranges; returns X, Q and the rr history (cap + 1, nsig)."""
    run = CG(nat, Ld, tau, a, d, B, cap)
    for it0, it1 in ranges:
        run.run(it0, it1)
    return run.X, run.Q, run.rr()


def cg_converged(nat, Ld, tau, a, d, B, stop, cap=2000):
    """Batches of 25 iterations until the relative residual of every column is below stop."""
    run, done = CG(nat, Ld, tau, a, d, B, cap), 0
    while done < cap:
        run.run(done, min(cap, done + 25))
        done = min(cap, done + 25)
        rr = run.scal[:(done + 1) * B.shape[1]].reshape(done + 1, -1).cpu().numpy()
        if np.all(rr[done] <= stop * stop * np.maximum(rr[0], 1e-300)):
            break
    return run.X


def scales(n, rng, kind, dt):
    """(row_scale, diag) device vectors and the labelled mask; at least one vertex labelled."""
    M = (rng.uniform(size=n) < 0.6).astype(F64)
    M[0] = 1
    if kind == "M":
        return None, dev(M, dt), np.ones(n), M
    if kind == "half":
        return None, dev(0.5 + M, dt), np.ones(n), 0.5 + M
    return dev(1 - M, dt), dev(M, dt), 1 - M, M


SCALES = ("M", "half", "constrained")
CG_NSIGS = (1, 2, 3, 5, 31, 32, 33, 64, 100, 128, 129, 200, 255, 256)


def check_solution(nat, L, n, nsig, kind, dt, tau, seed):
    rng = np.random.default_rng(seed)
    Ld = DeviceL(L, dt)
    a_d, d_d, a, d = scales(n, rng, kind, dt)
    B = rng.standard_normal((n, nsig))
    if kind == "constrained":
        B[d > 0] = 0                            # the right-hand side is zero on labelled rows
    A = (sparse.diags(a) @ (tau * L) + sparse.diags(d)).tocsc()
    ref = sla.spsolve(A, B).reshape(n, nsig)
    tol = 1e-8 if dt == F64 else 5e-5
    X = host(cg_converged(nat, Ld, tau, a_d, d_d, dev(B, dt), 1e-13 if dt == F64 else 1e-7))
    err = np.abs(X - ref).max(axis=0)
    scale = np.maximum(np.abs(ref).max(axis=0), 1e-300)
    assert np.all(err <= tol * scale), (n, nsig, kind, (err / scale).max())
    if kind == "constrained":
        assert np.all(X[d > 0] == 0)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("nsig", CG_NSIGS)
def test_cg_solves_every_width(gsp, nat, nsig, dt):
    """Lane shapes cw = 1 .. 256 against a float64 direct solve, on graphs smaller than, equal
    to and just over one CTA's rows."""
    for n in (1, 3, 255, 256, 257):
        L = banded_laplacian(n, n)
        for kind in SCALES:
            check_solution(nat, L, n, nsig, kind, dt, 1.5, n * 1000 + nsig)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("nsig", [1, 255, 256])
def test_cg_grid_at_the_block_cap(gsp, nat, sms, nsig, dt):
    """ceil(n / rows per pass) = 4 SM - 1, 4 SM and 4 SM + 1: at the last the grid is capped at
    4 SM CTAs, which then stride."""
    cw = 1
    while cw < nsig:
        cw *= 2
    rpb = 256 // cw
    for g in (4 * sms - 1, 4 * sms, 4 * sms + 1):
        n = rpb * (g - 1) + 1
        L = banded_laplacian(n, g)
        for kind in SCALES:
            check_solution(nat, L, n, nsig, kind, dt, 1.0, g)


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("nsig", [1, 33, 256])
def test_cg_first_iteration_is_exact(gsp, nat, sms, nsig, dt):
    """Integer L, tau, B and 0/1 scales: rr[0] = ||b||^2 and Q = tau L B (scaled) exactly, and
    X after one iteration is T(alpha b) with alpha = rr[0] / pq one float64 division."""
    rpb = 256 // (1 if nsig == 1 else (64 if nsig == 33 else 256))
    for n in (1, 3, 257, rpb * 4 * sms + 1):
        L = banded_laplacian(n, n)
        Ld = DeviceL(L, dt)
        Li = L.astype(np.int64)
        for kind in ("M", "constrained"):
            for tau in (1, 2):
                rng = np.random.default_rng(n + tau)
                a_d, d_d, a, d = scales(n, rng, kind, dt)
                B = rng.integers(-4, 5, size=(n, nsig)).astype(np.int64)
                if kind == "constrained":
                    B[d > 0] = 0
                X, Q, rr = cg(nat, Ld, tau, a_d, d_d, dev(B, dt), [(0, 1)], 1)
                Qx = a.astype(np.int64)[:, None] * (tau * (Li @ B)) + d.astype(np.int64)[:, None] * B
                assert_bits(host(Q), Qx)
                rr0 = (B * B).sum(axis=0)
                pq = (B * Qx).sum(axis=0)
                assert_bits(rr[0], rr0)
                alpha = np.where(pq > 0, rr0.astype(F64) / np.maximum(pq, 1).astype(F64), 0.0)
                assert_bits(host(X), (alpha[None, :] * B.astype(F64)).astype(dt))


@pytest.mark.parametrize("dt", [F64, F32])
@pytest.mark.parametrize("nsig", [1, 33, 256])
def test_cg_batches_and_special_columns(gsp, nat, sms, nsig, dt):
    """[0, 20) in one call, in batches of 1 and of 7: same X and rr history; a zero column stays
    exactly zero, a column solved in one step stays solved, and a second run repeats the bits."""
    import torch
    for n in (257, 5000):
        L = banded_laplacian(n, 7)
        Ld = DeviceL(L, dt)
        rng = np.random.default_rng(n + nsig)
        B = rng.standard_normal((n, nsig))
        zero, one = (0, nsig - 1) if nsig > 1 else (None, 0)
        if zero is not None:
            B[:, zero] = 0
        B[:, one] = 1
        Bd = dev(B, dt)
        ones = torch.ones(n, dtype=tdtype(dt), device="cuda")    # (tau L + I) 1 = 1
        k = 20
        X, _, rr = cg(nat, Ld, 1.5, None, ones, Bd, [(0, k)], k)
        for ranges in ([(i, i + 1) for i in range(k)], [(0, 7), (7, 14), (14, 20)]):
            Xb, _, rrb = cg(nat, Ld, 1.5, None, ones, Bd, ranges, k)
            assert_bits(host(Xb), host(X))
            assert_bits(rrb, rr)
        X2, _, rr2 = cg(nat, Ld, 1.5, None, ones, Bd, [(0, k)], k)
        assert_bits(host(X2), host(X))
        assert_bits(rr2, rr)
        Xh = host(X)
        assert not np.isnan(Xh).any() and not np.isnan(rr).any()
        if zero is not None:
            assert np.all(Xh[:, zero] == 0) and np.all(rr[:, zero] == 0)
        assert np.all(Xh[:, one] == 1) and np.all(rr[1:, one] == 0)
        if nsig > 2:
            assert np.all(rr[k, 1:nsig - 1] < rr[0, 1:nsig - 1])     # the others iterate


def test_cg_refuses_before_any_launch(gsp, nat):
    import torch
    L = banded_laplacian(100, 0)
    Ld = DeviceL(L, F64)
    before = nat.lib().gsp_launch_count()
    B = torch.zeros((100, 257), dtype=torch.float64, device="cuda")
    with pytest.raises(nat.NativeError, match="256"):
        cg(nat, Ld, 1.0, None, None, B, [(0, 1)], 1)
    B = B[:, :8].contiguous()
    for ranges, cap in (([(0, 3)], 2), ([(2, 1)], 5), ([(-1, 1)], 5)):
        with pytest.raises(nat.NativeError, match="iteration range"):
            cg(nat, Ld, 1.0, None, None, B, ranges, cap)
    assert nat.lib().gsp_launch_count() == before


# ----------------------------------------------------------------------------- FISTA last block
def fista_sizes(rpb, sms):
    """Row counts whose pass_blocks grid is 1, 2, 4 SM - 1, 4 SM and 4 SM + 1 (capped)."""
    return [rpb * g for g in (1, 2, 4 * sms - 1, 4 * sms)] + [rpb * 4 * sms + 1]


def relmax(a, b):
    return np.abs(np.asarray(a, dtype=np.float64) - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("C", [1, 3, 33])
def test_simplex_last_block_grids(gsp, sms, C):
    w = 1
    while w < min(C, 32):
        w *= 2
    runs = {}
    for n in fista_sizes(256 // w, sms):
        L, W = banded_laplacian(n, n), banded_adjacency(n, n)
        rng = np.random.default_rng(n)
        y = rng.integers(0, C, n).astype(F64)
        y[0] = C - 1
        M = rng.uniform(size=n) < 0.5
        M[0] = True
        lmax = 2.0 * L.diagonal().max() if n > 1 else 1.0
        for maxit in (1, 2, 17):
            ref, _, _, obj = lo.solve(L, y, M, 0.5, lmax, rtol=None, maxit=maxit)
            for dt, tol in ((F64, 1e-10), (F32, 1e-4)):
                G = gsp.graphs.Graph(W, dtype=dt)
                G._lmax, G._lmax_method = lmax, "lanczos"
                X = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=0.5, rtol=None,
                                                                 maxit=maxit, verbosity="NONE")
                rec = gsp.learning.last_solve
                assert (rec["niter"], rec["crit"]) == (maxit, "MAXIT")
                assert relmax(X, ref) <= tol, (n, maxit, dt)
                if dt == F64:
                    assert relmax(rec["objective"], obj) <= 1e-10
                runs[n, maxit, dt] = (G, y, M, X, rec["objective"])
    # every run again, each right after a run on another grid: the same bits
    for (n, maxit, dt), (G, y, M, X, obj) in sorted(runs.items(),
                                                    key=lambda kv: (kv[0][1], str(kv[0][2]), kv[0][0])):
        X2 = gsp.learning.classification_tikhonov_simplex(G, y, M, tau=0.5, rtol=None,
                                                          maxit=maxit, verbosity="NONE")
        assert_bits(X2, X)
        assert_bits(gsp.learning.last_solve["objective"], obj)


@pytest.mark.parametrize("nsig", [1, 3])
def test_prox_tv_last_block_grids(gsp, sms, nsig):
    """Both paths (the fused vertex pass, and A / At given) on paths of n vertices, n - 1 edges."""
    w = 1
    while w < nsig:
        w *= 2
    runs = {}
    ident = (lambda v: v)
    for n in fista_sizes(256 // w, sms):
        rng = np.random.default_rng(n)
        Wt = sparse.triu(sparse.diags([rng.uniform(0.5, 1.5, n - 1)], [1], shape=(n, n)))
        W = (Wt + Wt.T).tocsr()
        D = do.differential_operator(W)
        lmax = 2.0 * float(np.asarray(W.sum(axis=1)).max())
        x = rng.normal(size=(n, nsig))
        for maxit in (1, 2, 17):
            ref = oo.prox_tv_fgp(x, 0.3, D, lmax, tol=0, maxit=maxit)
            for dt in (F64, F32):
                G = gsp.graphs.Graph(W, dtype=dt)
                G._lmax, G._lmax_method = lmax, "lanczos"
                G.compute_differential_operator()
                for fused in (True, False):
                    kw = {} if fused else dict(A=ident, At=ident)
                    z = gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=maxit, **kw)
                    rec = gsp.optimization.last_solve
                    assert (rec["niter"], rec["crit"]) == (maxit, "MAXIT")
                    if dt == F64:
                        assert np.abs(z - ref["z"]).max() <= oo.F64_Z * np.abs(x).max()
                        for key in ("objective", "gap"):
                            assert (np.abs(rec[key] - ref[key]).max()
                                    <= oo.F64_HIST * np.abs(ref[key]).max())
                    else:
                        assert np.abs(z - ref["z"]).max() <= oo.F32_Z * np.abs(x).max()
                    runs[n, maxit, dt, fused] = (G, x, kw, z, rec["objective"])
    for (n, maxit, dt, fused), (G, x, kw, z, obj) in sorted(
            runs.items(), key=lambda kv: (kv[0][1], str(kv[0][2]), kv[0][3], kv[0][0])):
        z2 = gsp.optimization.prox_tv(x, 0.3, G, tol=0, maxit=maxit, **kw)
        assert_bits(z2, z)
        assert_bits(gsp.optimization.last_solve["objective"], obj)


# ------------------------------------------------------------------------- beyond 2^31 elements
def test_reductions_beyond_2_31_elements(gsp, nat):
    """An (2^24 + 3, 128) float32 block, 2^31 + 384 elements, as both operands of the moments
    pass and block_residual, against closed-form per-column counts."""
    import torch
    from pygsp_b200.graphs import fourier as fr
    free, _ = torch.cuda.mem_get_info()
    if free < 12 * 2**30:
        pytest.skip("needs 12 GB of free device memory, %.1f GB free" % (free / 2**30))
    n, b = 2**24 + 3, 128
    X = torch.empty((n, b), dtype=torch.float32, device="cuda")
    j = torch.arange(b, device="cuda")
    step = 2**20
    for r0 in range(0, n, step):
        r = torch.arange(r0, min(n, r0 + step), device="cuda")[:, None]
        X[r0:r0 + step] = ((7 * r + j) % 5 - 2).float()
    # (7 r + j) mod 5 = (2 r' + j) mod 5 for r = 5 q + r': each residue q times, plus the first s
    q, s = divmod(n, 5)
    ref = np.empty(b)
    for c in range(b):
        count = np.full(5, q)
        for rp in range(s):
            count[(2 * rp + c) % 5] += 1
        ref[c] = float((count * (np.arange(5) - 2) ** 2).sum())
    mom = host(moments(nat, X, X)[0])
    assert_bits(mom, np.stack([ref, ref]))
    theta = np.full(b, 3.0)                      # (X - 3 X)^2 = 4 X^2
    assert_bits(fr.block_residual(X, X, theta), 4 * ref)
    del X
    torch.cuda.empty_cache()
