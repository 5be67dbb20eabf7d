"""The one dispatch of a Chebyshev step between the TMA-tiled and the row-group kernel.

The tiled kernel issues 16-byte TMA copies and float4 loads, so a step takes it only when every
block it touches is 16-byte aligned (and a tile plan applies).  Without a halo a step that fails
that test runs on the row-group kernel; with a halo it is refused, because the row-group kernel
neither waits for the neighbours nor pushes or publishes.  Single-GPU and partitioned calls run
the same coefficient schedule through the same dispatch, so they give the same bits.
"""
import ctypes

import numpy as np
import pytest
from scipy import sparse

from oracle import pygsp_oracle as orc
from oracle import step_oracle as so

NAN32 = 0x7FE5A5A5                 # quiet NaN with a payload: rows a step must not touch
BLOCKS = ("x_cur", "x_new", "r", "indptr", "indices", "data")


@pytest.mark.parametrize("misaligned", BLOCKS + (None,))
def test_halo_step_refuses_unaligned_blocks_without_a_launch(misaligned):
    """Fake device addresses, one of them 4 bytes off a 16-byte boundary: the halo step returns
    GSP_ERR_UNSUPPORTED before any CUDA call.  With every block aligned it gets as far as the
    launch, which fails on a machine without a device."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("passes fake device pointers: CPU only")
    from pygsp_b200 import _native as nat
    addr = {name: 0x7F0000000000 + (i << 24) for i, name in enumerate(BLOCKS + ("x_old",))}
    if misaligned:
        addr[misaligned] += 4
    p = lambda name: ctypes.c_void_p(addr[name])
    plan = nat.TilePlan(rows_per_tile=64, slab_capacity=1024, stages=2, consumer_warps=16,
                        gather_unroll=4, blocks_per_sm=0)
    expect = r"\(-3\): fused halo step: the tiled kernel does not apply" if misaligned else r"\(-2\)"
    with pytest.raises(nat.NativeError, match=expect):
        nat.call("gsp_cheby_step_halo_f32", nat.i32(0), nat.i64(1000), nat.i64(8000), p("indptr"),
                 p("indices"), p("data"), p("x_cur"), p("x_old"), p("x_new"), p("r"),
                 nat.i64(1000), nat.i64(64), nat.i32(1), np.ones(1), np.ones(1), nat.f64(0.5),
                 nat.f64(-2.0), nat.f64(-1.0), nat.i32(0), plan, nat.HaloFusion(), None)


def _sentinel(torch, count):
    return torch.full((count,), NAN32, dtype=torch.int32, device="cuda").view(torch.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("first", [True, False])
def test_unaligned_step_equals_the_tiled_step(first):
    """gsp_cheby_step_f32 with a tile plan on x_cur, x_new and r that start one float past a
    16-byte boundary runs on the row-group kernel alone and returns the tiled step's bits on the
    same data; rows outside [rb, n) keep their contents."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import pygsp_b200 as gsp
    from pygsp_b200 import _native as nat
    nsig, rb = 64, 8
    n = rb + 300 * 64 + 5
    W = so.sensor_adjacency(n, k=8, seed=11)
    L = orc.laplacian(sparse.csr_matrix(W)).astype(np.float32)
    L.eliminate_zeros()
    L.sort_indices()
    lmax = 1.01 * float(abs(L.astype(np.float64)).sum(axis=1).max())
    dev = gsp.graphs.DeviceCSR.from_scipy(L, torch.float32, torch.device("cuda"))
    plan = dev.tile_plan(nsig, 1)
    assert plan is not None and plan.rows_per_tile == 64
    rng = np.random.default_rng(first)
    xc = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()
    xo = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()
    r_old = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()
    ck, c0 = rng.standard_normal(1), rng.standard_normal(1)
    r_rows = n + 12
    count = nat.lib().gsp_launch_count
    count.restype = ctypes.c_uint64

    def run(offset):
        x_cur = _sentinel(torch, n * nsig + offset)[offset:].view(n, nsig)
        x_new = _sentinel(torch, n * nsig + offset)[offset:].view(n, nsig)
        r = _sentinel(torch, r_rows * nsig + offset)[offset:].view(r_rows, nsig)
        assert (x_cur.data_ptr() % 16 == 0) == (offset == 0)
        x_cur.copy_(xc)
        if not first:
            r[rb:n] = r_old[rb:]
        launches = count()
        nat.call("gsp_cheby_step_f32", nat.i32(int(first)), nat.i64(rb), nat.i64(n),
                 nat.i64(dev.nnz), dev.indptr, dev.indices, dev.data, x_cur,
                 None if first else xo, x_new, r, nat.i64(r_rows), nat.i64(nsig), nat.i32(1),
                 ck, c0, nat.f64(3.7 / lmax), nat.f64(-1.93), nat.f64(0.0 if first else -0.87),
                 plan, nat.stream_ptr(dev.device))
        torch.cuda.synchronize()
        return x_new.view(torch.int32).cpu(), r.view(torch.int32).cpu(), count() - launches

    x_al, r_al, k_al = run(0)
    x_un, r_un, k_un = run(1)
    assert (k_al, k_un) == (2, 1)           # tiled + remainder rows; row-group kernel only
    assert torch.equal(x_un, x_al)
    assert torch.equal(r_un, r_al)
    assert (x_un[:rb] == NAN32).all() and (r_un[:rb] == NAN32).all() and (r_un[n:] == NAN32).all()


@pytest.mark.gpu
def test_partitioned_single_rank_clenshaw_matches_graph_path():
    """One filter of order 15 on a single-rank PartitionedCheby: the partitioned call's Clenshaw
    recurrence (csrc/dist.cu) against gsp_cheby_clenshaw_f32 on the whole graph, bit for bit."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import torch.distributed as dist
    import pygsp_b200 as gsp
    from pygsp_b200 import distributed as gd
    from pygsp_b200.filters import approximations as apx
    G = gsp.graphs.Sensor(20000, k=8, seed=3, order="morton")
    G.estimate_lmax()
    plan = gd.HaloPlan(G.L.to_scipy(), gd.even_bounds(G.N, 1), 0)
    c = np.random.default_rng(1).standard_normal((1, 16)) / np.arange(1, 17)
    x = torch.randn(G.N, 64, device="cuda")
    # the peer window exchanges its IPC handle once: a one-process group in memory
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        op = gd.PartitionedCheby(plan, exchange="p2p")
        a = op.cheby_op(G.lmax, c, x)
        torch.cuda.synchronize()
        for w in op._windows.values():
            w.close()
    finally:
        dist.destroy_process_group()
    b = apx.cheby_clenshaw_device(G.L, G.lmax, c, x)
    assert a.shape == (1, G.N, 64)
    assert torch.equal(a[0], b)
