"""How the tiled Chebyshev step (csrc/cheby_tiled.cu) hands its row tiles to persistent CTAs.

Single steps are run at tile counts on both sides of the grid size (fewer tiles than the grid
could hold, grid - 1, grid, grid + 1, a count that is not a multiple of the grid), with the
row range starting at row 0 and further in, walking the tiles in both directions, and every row
of the range is checked against the float64 step of oracle/step_oracle.py within its proven
bound; rows outside the range must come back bit-unchanged.  Whole forward and Clenshaw calls at
the same tile counts must equal the row-group kernel bit for bit.  The grid is known exactly
with one CTA per SM (GSPB200_TILE_BPS=1: min(tiles, SMs)); the default launch is covered too.
"""
import numpy as np
import pytest
from scipy import sparse

from conftest import relerr_cols
from oracle import pygsp_oracle as orc
from oracle import step_oracle as so

pytestmark = pytest.mark.gpu

NAN32 = 0x7FE5A5A5                 # quiet NaN with a payload: rows a step must not touch
TAIL = 5                           # rows past the last full tile (row-group kernel)


@pytest.fixture(scope="module")
def env():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200, torch.cuda.get_device_properties(0).multi_processor_count


def _graph(gsp, n, seed):
    import torch
    W = so.sensor_adjacency(n, k=8, seed=seed)
    L = orc.laplacian(sparse.csr_matrix(W)).astype(np.float32)
    L.eliminate_zeros()
    L.sort_indices()
    lmax = 1.01 * float(abs(L.astype(np.float64)).sum(axis=1).max())
    return L, gsp.graphs.DeviceCSR.from_scipy(L, torch.float32, torch.device("cuda")), lmax


def _plan(dev, nsig, monkeypatch, bps):
    """Plan with at most `bps` CTAs per SM (1: the grid is min(tiles, SMs), known exactly)."""
    monkeypatch.setenv("GSPB200_TILE_BPS", str(bps))
    dev._plans.clear()
    plan = dev.tile_plan(nsig, 1)
    dev._plans.clear()
    assert plan is not None and plan.blocks_per_sm == bps
    return plan


def _tile_rows(nsig):
    """Rows per tile of the default plan for one filter."""
    return 256 if nsig == 8 else (32 if nsig == 128 else 64)


def _sentinel(torch, shape):
    return torch.full(shape, NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


def _step(gsp, L, dev, lmax, plan, nsig, first, rb, reverse, seed):
    """One step over [rb, n) into NaN-filled x_new / r: every row in range within the oracle's
    bound, every element out of range bit-unchanged.  reverse=None: gsp_cheby_step_f32 (forward
    walk); True / False: gsp_cheby_step_halo_f32 with no neighbours (rows [0, n), that direction)."""
    import torch
    from pygsp_b200 import _native as nat
    n = L.shape[0]
    rng = np.random.default_rng(seed)
    xc = so.scaled_signals(rng, n, nsig)
    xo = so.scaled_signals(rng, n, nsig)
    r_old = so.scaled_signals(rng, n, nsig)[None]
    ck = np.ascontiguousarray(rng.standard_normal(1))
    c0 = np.ascontiguousarray(rng.standard_normal(1))
    a, b, g = 3.7 / lmax, -1.93, (0.0 if first else -0.87)
    ref_x, ref_r, bx, br = so.step_reference(L, xc, xo, r_old, a, b, g, ck, c0, first)
    r_rows = n + 12
    r_buf = _sentinel(torch, (1, r_rows, nsig))
    if not first:
        r_buf[0, rb:n] = torch.from_numpy(r_old[0, rb:n]).cuda()
    xn = _sentinel(torch, (n, nsig))
    x_before, r_before = xn.view(torch.int32).cpu(), r_buf.view(torch.int32).cpu()
    xc_d, xo_d = torch.from_numpy(xc).cuda(), torch.from_numpy(xo).cuda()
    common = (dev.indptr, dev.indices, dev.data, xc_d, None if first else xo_d, xn, r_buf,
              nat.i64(r_rows), nat.i64(nsig), nat.i32(1), ck, c0, nat.f64(a), nat.f64(b), nat.f64(g))
    if reverse is None:
        nat.call("gsp_cheby_step_f32", nat.i32(int(first)), nat.i64(rb), nat.i64(n),
                 nat.i64(dev.nnz), *common, plan, nat.stream_ptr(dev.device))
    else:
        assert rb == 0
        nat.call("gsp_cheby_step_halo_f32", nat.i32(int(first)), nat.i64(n), nat.i64(dev.nnz),
                 *common, nat.i32(int(reverse)), plan, nat.HaloFusion(), nat.stream_ptr(dev.device))
    torch.cuda.synchronize()
    what = "nsig=%d first=%d rows [%d, %d) reverse=%s" % (nsig, first, rb, n, reverse)
    x_after, r_after = xn.view(torch.int32).cpu(), r_buf.view(torch.int32).cpu()
    assert torch.equal(x_after[:rb], x_before[:rb]), what + " (x_new before the range)"
    assert torch.equal(r_after[0, :rb], r_before[0, :rb]), what + " (r before the range)"
    assert torch.equal(r_after[0, n:], r_before[0, n:]), what + " (r past the range)"
    got_x = xn[rb:].cpu().numpy()
    got_r = r_buf[0, rb:n].cpu().numpy()
    bad_x = so.violations(got_x, ref_x[rb:], bx[rb:])
    bad_r = so.violations(got_r, ref_r[0, rb:], br[0, rb:])
    assert not bad_x.any(), (what + " x_new", rb + np.argwhere(bad_x)[0][0], int(bad_x.sum()))
    assert not bad_r.any(), (what + " r", rb + np.argwhere(bad_r)[0][0], int(bad_r.sum()))


def _tile_counts(sms):
    """Tile counts of a launch with one CTA per SM (grid = min(tiles, SMs))."""
    return (5, sms - 1, sms, sms + 1, 2 * sms + sms // 2 + 1)


@pytest.mark.parametrize("nsig", [8, 64, 128])
def test_single_steps_at_tile_counts_around_the_grid(env, monkeypatch, nsig):
    gsp, sms = env
    R = _tile_rows(nsig)
    for k, tiles in enumerate(_tile_counts(sms)):
        rb = 4 * (3 + k) if k % 2 else 0                 # rb > 0 on every other count
        n = rb + tiles * R + TAIL
        L, dev, lmax = _graph(gsp, n, seed=tiles)
        plan = _plan(dev, nsig, monkeypatch, 1)
        assert plan.rows_per_tile == R and (n - rb) // R == tiles
        for first in (True, False):
            _step(gsp, L, dev, lmax, plan, nsig, first, rb, None, seed=tiles + first)
        if rb == 0:
            for reverse in (False, True):
                _step(gsp, L, dev, lmax, plan, nsig, False, 0, reverse, seed=tiles + 7)


@pytest.mark.parametrize("nsig", [8, 64, 128])
def test_single_steps_with_every_cta_of_the_sm(env, monkeypatch, nsig):
    """As many CTAs per SM as fit (the default launch): a count that is no multiple of the grid,
    staged and direct vectors, both directions."""
    gsp, sms = env
    R = _tile_rows(nsig)
    tiles = 7 * sms + 3
    n = tiles * R + TAIL
    L, dev, lmax = _graph(gsp, n, seed=nsig)
    plan = _plan(dev, nsig, monkeypatch, 0)
    for vdir in ("0", "1"):
        monkeypatch.setenv("GSPB200_TILE_VDIR", vdir)
        _step(gsp, L, dev, lmax, plan, nsig, False, 64, None, seed=1)
        for reverse in (False, True):
            _step(gsp, L, dev, lmax, plan, nsig, False, 0, reverse, seed=2 + reverse)


def _calls(gsp, dev, lmax, c, x, src):
    import torch
    from pygsp_b200.filters import approximations as apx
    fwd = apx.cheby_op_device(dev, lmax, c, x)
    cl = apx.cheby_clenshaw_device(dev, lmax, c, src)
    torch.cuda.synchronize()
    return fwd.clone(), cl.clone()


@pytest.mark.parametrize("nsig", [8, 64, 128])
def test_whole_calls_equal_the_row_group_kernel(env, monkeypatch, nsig):
    """Forward and Clenshaw calls (every other step walks the tiles backwards) at the tile counts
    above, with one CTA per SM and with the default launch: the row-group kernel's bits, and
    within 1e-5 of the float64 oracle."""
    import torch
    gsp, sms = env
    R = _tile_rows(nsig)
    rng = np.random.default_rng(nsig)
    for tiles in _tile_counts(sms)[1:]:
        n = tiles * R + TAIL
        L, dev, lmax = _graph(gsp, n, seed=tiles)
        x = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()
        src = torch.from_numpy(so.scaled_signals(rng, n, nsig)[None]).cuda()
        c = rng.standard_normal((1, 13)) / np.arange(1, 14) ** 2
        with monkeypatch.context() as m:
            m.setenv("GSPB200_KERNEL", "rowgroup")
            dev._plans.clear()
            assert dev.tile_plan(nsig, 1) is None
            want = _calls(gsp, dev, lmax, c, x, src)
        for bps in (1, 0):
            _plan(dev, nsig, monkeypatch, bps)
            got = _calls(gsp, dev, lmax, c, x, src)
            dev._plans.clear()
            for form, a, b in zip(("forward", "Clenshaw"), got, want):
                assert torch.equal(a, b), (form, nsig, tiles, bps, int((a != b).sum()))
        Lo = L.astype(np.float64)
        ref = orc.cheby_op(Lo, lmax, c, x[:, :2].double().cpu().numpy())
        assert relerr_cols(want[0][:, :, :2].reshape(n, -1).cpu().numpy(), ref) <= 1e-5
        ref = orc.cheby_op(Lo, lmax, c[0], src[0][:, :2].double().cpu().numpy())
        assert relerr_cols(want[1][:, :2].cpu().numpy(), ref) <= 1e-5
