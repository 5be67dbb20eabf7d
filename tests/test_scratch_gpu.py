"""Stream-ordered device scratch of the C entry points (gsp::Scratch, gsp::cub_temp in
csrc/common.cuh) is released on every return: each entry point that allocates scratch runs on
small inputs through its public Python caller, and afterwards the memory in use in the device's
default memory pool -- the pool cudaMallocAsync draws from -- is back where it started.  The
input-error return of the COO conversion, taken after its buffers are allocated, is checked the
same way."""
import ctypes

import numpy as np
import pytest
from scipy import sparse

pytestmark = pytest.mark.gpu

CU_MEMPOOL_ATTR_USED_MEM_CURRENT = 7          # cuda.h, enum CUmemPool_attribute


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if torch.cuda.get_allocator_backend() == "cudaMallocAsync":
        pytest.skip("torch's own blocks would share the default memory pool")
    import pygsp_b200
    return pygsp_b200


@pytest.fixture(scope="module")
def pool_used(gsp):
    """Bytes in use in the current device's default memory pool, after a synchronise."""
    import torch
    torch.zeros(1, device="cuda")                           # the primary context exists
    cuda = ctypes.CDLL("libcuda.so.1")
    dev = ctypes.c_int()
    assert cuda.cuDeviceGet(ctypes.byref(dev), torch.cuda.current_device()) == 0
    pool = ctypes.c_void_p()
    assert cuda.cuDeviceGetDefaultMemPool(ctypes.byref(pool), dev) == 0

    def used():
        torch.cuda.synchronize()
        value = ctypes.c_uint64()
        assert cuda.cuMemPoolGetAttribute(pool, CU_MEMPOOL_ATTR_USED_MEM_CURRENT,
                                          ctypes.byref(value)) == 0
        return value.value
    return used


def _ring(n):
    i = np.arange(n)
    return sparse.csr_matrix((np.ones(2 * n), (np.r_[i, i], np.r_[(i + 1) % n, (i - 1) % n])),
                             shape=(n, n))


def _star(leaves):
    """Hub row with more two-hop candidates than a row counted in shared memory."""
    n = leaves + 1
    rows = np.r_[np.zeros(leaves, dtype=int), np.arange(1, n)]
    cols = np.r_[np.arange(1, n), np.zeros(leaves, dtype=int)]
    return sparse.csr_matrix((np.ones(2 * leaves), (rows, cols)), shape=(n, n))


def graph_from_coo(gsp):
    import torch
    rng = np.random.default_rng(0)
    rows = torch.as_tensor(rng.integers(0, 200, 1000), device="cuda")
    cols = torch.as_tensor(rng.integers(0, 200, 1000), device="cuda")
    vals = torch.ones(1000, dtype=torch.float64, device="cuda")
    G = gsp.graphs.Graph.from_coo(rows, cols, vals, 200)
    assert G.W.nnz <= 1000


def directed_transpose(gsp):
    W = sparse.triu(sparse.random(300, 300, density=0.02, random_state=1), k=1).tocsr()
    G = gsp.graphs.Graph(W, dtype=np.float64)
    assert G.is_directed()
    assert G._transpose().nnz == W.nnz


def knn_cell_grid(gsp):
    gsp.graphs.Sensor(500, k=6, seed=1)
    gsp.graphs.NNGraph(np.random.default_rng(2).uniform(size=(400, 3)), k=5)


def components_and_subgraph(gsp):
    G = gsp.graphs.Graph(sparse.block_diag([_ring(30), _ring(20)]).tocsr(), dtype=np.float64)
    assert [C.N for C in G.extract_components()] == [30, 20]
    assert G.subgraph([40, 3, 7, 35]).N == 4


def sparsify(gsp):
    G = gsp.graphs.Sensor(3000, k=10, seed=6, dtype=np.float64, order="morton")
    gsp.reduction.graph_sparsify(G, 0.3, seed=11)


def two_hop_count(gsp):
    gsp.features.compute_avg_adj_deg(gsp.graphs.Graph(_star(2000), dtype=np.float32))


def moments(gsp):
    G = gsp.graphs.Sensor(300, k=6, seed=4, dtype=np.float64)
    gsp.features.compute_norm_tig(gsp.filters.Heat(G, scale=10), order=20)


def lanczos(gsp):
    x = np.random.default_rng(5).normal(size=(400, 3))
    gsp.filters.lanczos(_ring(400).astype(np.float64), 12, x)


def fourier_blocks(gsp):
    import torch
    from pygsp_b200.graphs import fourier
    for n in (100, 20000):                       # one partition, several partitions
        X = torch.randn(n, 8, dtype=torch.float64, device="cuda")
        LX = torch.randn(n, 8, dtype=torch.float64, device="cuda")
        fourier.block_gram(X, LX)
        fourier.block_residual(X, LX, np.linspace(0, 1, 8))


def tile_plan(gsp):
    G = gsp.graphs.Sensor(2000, k=6, seed=7, order="morton", dtype=np.float32)
    assert G.L.tile_plan(32, 0) is not None


CASES = [graph_from_coo, directed_transpose, knn_cell_grid, components_and_subgraph, sparsify,
         two_hop_count, moments, lanczos, fourier_blocks, tile_plan]


@pytest.mark.parametrize("case", CASES, ids=[c.__name__ for c in CASES])
def test_scratch_released(gsp, pool_used, case):
    before = pool_used()
    case(gsp)
    assert pool_used() == before


def test_scratch_released_on_out_of_range_coo(gsp, pool_used):
    import torch
    from pygsp_b200 import _native as nat
    n, nnz = 50, 40
    rows = torch.arange(nnz, dtype=torch.int32, device="cuda")
    cols = rows.clone()
    cols[7] = n                                              # one column out of range
    vals = torch.ones(nnz, dtype=torch.float64, device="cuda")
    indptr = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    indices = torch.empty(nnz, dtype=torch.int32, device="cuda")
    data = torch.empty(nnz, dtype=torch.float64, device="cuda")
    uniq = ctypes.c_int64(0)
    before = pool_used()
    with pytest.raises(nat.NativeError, match="out of range"):
        nat.call("gsp_coo_to_csr_f64", nat.i64(n), nat.i64(nnz), rows, cols, vals, indptr,
                 indices, data, ctypes.byref(uniq), nat.stream_ptr())
    assert pool_used() == before
