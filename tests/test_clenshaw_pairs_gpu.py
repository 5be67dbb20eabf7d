"""Clenshaw filtering with the middle steps run two per launch (cheby_pair_tiled).

A paired call must give the bits of the single-step call: every tiled width, orders with no
pair, one pair, a left-over middle step and many pairs, graphs with rows past the last full tile,
with a structure that is not symmetric, with scattered gathers, and a 2^18-row Morton k-NN graph
on which every CTA walks many slots and the selection by block size pairs on its own.
"""
import numpy as np
import pytest

from conftest import relerr_cols
from oracle import pygsp_oracle as orc
from oracle import step_oracle as so

pytestmark = pytest.mark.gpu

F32_TOL = 1e-5
ORDERS = (2, 3, 4, 5, 30, 31)


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200
    return pygsp_b200


def _laplacian32(W):
    L = orc.laplacian(W.tocsr()).astype(np.float32)
    L.sort_indices()
    return L


def _graphs():
    rng = np.random.default_rng(11)
    base = so.sensor_adjacency(4096, k=8, seed=21)
    p = rng.permutation(4096)
    D = base.copy()
    D.data = D.data * (rng.uniform(size=D.nnz) > 0.2)
    D.eliminate_zeros()
    assert orc.is_directed(D)
    return {"morton k-NN": _laplacian32(base),
            "rows past the last tile": _laplacian32(so.sensor_adjacency(4096 + 37, k=8, seed=22)),
            "renumbered": _laplacian32(base[p][:, p]),
            "one-way edges": _laplacian32(D)}


def _run(monkeypatch, apx, dev, lmax, c, x, pairs, **kw):
    """(result, kernels launched) of one call; the plans are built by a call before the count."""
    import torch
    lib = __import__("pygsp_b200")._native.lib()
    with monkeypatch.context() as m:
        if pairs is not None:
            m.setenv("GSPB200_CLENSHAW_PAIRS", pairs)
        apx.cheby_clenshaw_device(dev, lmax, c, x, **kw)
        before = lib.gsp_launch_count()
        out = apx.cheby_clenshaw_device(dev, lmax, c, x, **kw)
        torch.cuda.synchronize()
        return out, lib.gsp_launch_count() - before


@pytest.mark.parametrize("name", ["morton k-NN", "rows past the last tile", "renumbered", "one-way edges"])
@pytest.mark.parametrize("lag", ["0", "3", None])
def test_pairs_give_the_bits_of_single_steps(gsp, monkeypatch, name, lag):
    import torch
    from pygsp_b200.filters import approximations as apx
    if lag is not None:
        monkeypatch.setenv("GSPB200_PAIR_LAG", lag)
    L = _graphs()[name]
    n = L.shape[0]
    lmax = 1.01 * float(abs(L.astype(np.float64)).sum(axis=1).max())
    dev = gsp.graphs.DeviceCSR.from_scipy(L, torch.float32, torch.device("cuda"))
    rng = np.random.default_rng(3)
    for nsig in (8, 16, 32, 64, 128):
        x = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()
        for order in ORDERS:
            c = rng.standard_normal(order + 1) / np.arange(1, order + 2) ** 2
            single, n_single = _run(monkeypatch, apx, dev, lmax, c, x, "0")
            paired, n_paired = _run(monkeypatch, apx, dev, lmax, c, x, "1")
            # two launches become one; with rows past the last tile, four become three
            assert n_single - n_paired == max(0, (order - 3) // 2), (nsig, order)
            assert torch.equal(single, paired), (name, nsig, order, int((single != paired).sum()))
            if order in (5, 30) and lag is None:
                ref = orc.cheby_op(L.astype(np.float64), lmax, c, x.double().cpu().numpy())
                assert relerr_cols(paired.cpu().numpy(), ref) <= F32_TOL


def test_large_graph_pairs_by_default(gsp, monkeypatch):
    """2^18 rows: 660 tiles per CTA at 64 signals; a 128-signal block (134 MB) exceeds L2, so the
    call pairs without being told to, and a caller's two-block work keeps single steps."""
    import torch
    from pygsp_b200.filters import approximations as apx
    G = gsp.graphs.Sensor(1 << 18, k=8, seed=7, order="morton")
    G.estimate_lmax()
    n = G.N
    rng = np.random.default_rng(4)
    for nsig, orders in ((128, (30, 31)), (64, (30,)), (8, (31,))):
        x = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()
        for order in orders:
            c = rng.standard_normal(order + 1) / np.arange(1, order + 2) ** 2
            single, n_single = _run(monkeypatch, apx, G.L, G.lmax, c, x, "0")
            paired, n_paired = _run(monkeypatch, apx, G.L, G.lmax, c, x, "1")
            assert n_single - n_paired == (order - 3) // 2
            assert torch.equal(single, paired), (nsig, order, int((single != paired).sum()))
            if nsig == 128:
                auto, n_auto = _run(monkeypatch, apx, G.L, G.lmax, c, x, None)
                assert n_auto == n_paired and torch.equal(auto, single)
                work = torch.empty((2, n, nsig), dtype=torch.float32, device="cuda")
                two, n_two = _run(monkeypatch, apx, G.L, G.lmax, c, x, None, work=work)
                assert n_two == n_single and torch.equal(two, single)
    Lh = G.L.to_scipy().astype(np.float64)
    ref = orc.cheby_op(Lh, G.lmax, c, x[:, :4].double().cpu().numpy())
    assert relerr_cols(paired[:, :4].cpu().numpy(), ref) <= F32_TOL
