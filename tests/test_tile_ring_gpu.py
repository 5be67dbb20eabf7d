"""Tiled Clenshaw steps that gather from each tile's neighbour ring in shared memory.

The ring changes where the gathered rows come from, not the sums: a call must give the bits of
the row-group kernel (GSPB200_KERNEL=rowgroup) and of the tiled kernel without rings
(GSPB200_TILE_RING=0), at every tiled width, for orders with no pair, one pair, a left-over middle
step and many pairs, with pairs on and off, on the graphs of the paired-launch tests (rows past
the last full tile, one-way edges) and on a 2^18-row Morton graph where every CTA walks many
slots.  A graph whose largest ring does not fit takes the kernel without rings, with the same bits.
"""
import ctypes

import numpy as np
import pytest

from oracle import step_oracle as so
from test_clenshaw_pairs_gpu import _graphs

pytestmark = pytest.mark.gpu

ORDERS = (2, 3, 5, 30, 31)
WIDTHS = (8, 16, 32, 64, 128)


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


def _call(monkeypatch, L, lmax, c, x, **env):
    import torch
    from pygsp_b200.filters import approximations as apx
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv("GSPB200_" + k, v)
        out = apx.cheby_clenshaw_device(L, lmax, c, x)
        torch.cuda.synchronize()
        return out


def _ring_fits(gsp, L, nsig):
    plan = L.tile_plan(nsig, 1)
    ring = L.ring_plan(plan.rows_per_tile) if plan is not None else None
    return ring is not None and bool(gsp._native.lib().gsp_cheby_ring_fits(
        ring.ring_max, gsp._native.i64(nsig), ctypes.byref(plan)))


def _check_bits(gsp, monkeypatch, Lh, lmax, dev, widths, orders, seed):
    """Ring, no ring and row-group calls give the same bits, pairs on and off."""
    import torch
    rowgroup = gsp.graphs.DeviceCSR.from_scipy(Lh, torch.float32, torch.device("cuda"))
    with monkeypatch.context() as m:
        m.setenv("GSPB200_KERNEL", "rowgroup")
        assert rowgroup.tile_plan(8, 1) is None
    rng = np.random.default_rng(seed)
    fits = {}
    for nsig in widths:
        x = torch.from_numpy(so.scaled_signals(rng, Lh.shape[0], nsig)).cuda()
        fits[nsig] = _ring_fits(gsp, dev, nsig)
        for order in orders:
            c = rng.standard_normal(order + 1) / np.arange(1, order + 2) ** 2
            ref = _call(monkeypatch, rowgroup, lmax, c, x, KERNEL="rowgroup")
            for pairs in ("0", "1"):
                off = _call(monkeypatch, dev, lmax, c, x, TILE_RING="0", CLENSHAW_PAIRS=pairs)
                on = _call(monkeypatch, dev, lmax, c, x, CLENSHAW_PAIRS=pairs)
                assert torch.equal(on, ref), (nsig, order, pairs, int((on != ref).sum()))
                assert torch.equal(on, off), (nsig, order, pairs)
    return fits


@pytest.mark.parametrize("name", ["morton k-NN", "rows past the last tile", "renumbered",
                                  "one-way edges"])
def test_ring_gives_the_bits_of_the_gather(gsp, monkeypatch, name):
    import torch
    Lh = _graphs()[name]
    lmax = 1.01 * float(abs(Lh.astype(np.float64)).sum(axis=1).max())
    dev = gsp.graphs.DeviceCSR.from_scipy(Lh, torch.float32, torch.device("cuda"))
    fits = _check_bits(gsp, monkeypatch, Lh, lmax, dev, WIDTHS, ORDERS, 5)
    if name == "renumbered":
        # scattered columns: the largest ring does not fit at 128 signals, the kernel without
        # rings runs (and gave the bits above)
        assert not fits[128]
    else:
        assert all(fits.values()), fits


def test_ring_on_a_large_graph(gsp, monkeypatch):
    """2^18 rows: hundreds of slots per CTA, single steps and pairs."""
    G = gsp.graphs.Sensor(1 << 18, k=8, seed=7, order="morton")
    G.estimate_lmax()
    Lh = G.L.to_scipy()
    fits = _check_bits(gsp, monkeypatch, Lh, G.lmax, G.L, (64, 128), (30, 31), 6)
    assert all(fits.values()), fits


def test_ring_that_does_not_fit(gsp, monkeypatch):
    """A tile whose ring is the whole graph: the plan reports that it does not fit, the call is
    the gather's, bit for bit; a ring exactly at the budget's edge is accepted."""
    import torch
    from scipy import sparse
    n = 8192
    path = sparse.diags([np.ones(n - 1)], [1], shape=(n, n))
    hub = sparse.lil_matrix((n, n))
    hub[100, :] = 1.0
    hub[100, 100] = 0.0
    W = (path + path.T + hub + hub.T).tocsr()
    Lh = (sparse.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr().astype(np.float32)
    Lh.sort_indices()
    dev = gsp.graphs.DeviceCSR.from_scipy(Lh, torch.float32, torch.device("cuda"))
    plan = dev.tile_plan(64, 1)
    ring = dev.ring_plan(plan.rows_per_tile)
    assert ring.ring_max == n
    lib = gsp._native.lib()
    assert not lib.gsp_cheby_ring_fits(ring.ring_max, gsp._native.i64(64), ctypes.byref(plan))
    # the largest ring that fits is accepted, one row more is not
    fit = max(r for r in range(1, n) if lib.gsp_cheby_ring_fits(r, gsp._native.i64(64),
                                                                ctypes.byref(plan)))
    assert 64 < fit < n
    lmax = 1.01 * float(abs(Lh.astype(np.float64)).sum(axis=1).max())
    _check_bits(gsp, monkeypatch, Lh, lmax, dev, (64,), (5, 30), 7)
