"""The count half of every CSR count / fill pair reports its number of entries one way: through
its ``int64_t* nnz`` argument, the int64 sum of the row sizes that ``gsp::scan_rows`` scans into
the int32 indptr.

On small matrices and graphs, empty ones included, the total equals indptr[-1], and a NULL total
leaves the indptr bytes as they are.  ``Grid2d(33600, 33600)`` holds 4 * 33600 * 33599 =
4 515 705 600 entries, which the int32 scan wraps to a positive 220 738 304: the count reports the
true total, and ``Grid2d`` refuses the graph before it allocates anything beyond indptr and the
total.  No fill runs here."""
import gc

import numpy as np
import pytest
from scipy import sparse

pytestmark = pytest.mark.gpu

SFX = ["f32", "f64"]
GRID = 33600
GRID_NNZ = 4 * GRID * (GRID - 1)


@pytest.fixture(scope="module")
def gsp():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import pygsp_b200
    return pygsp_b200


def counted(gsp, name, n, *args):
    """Run count entry point ``name(*args, indptr, nnz, stream)`` for an indptr of n + 1 entries,
    once with a total and once with NULL; check that the total is indptr[-1] and that both
    indptr agree byte for byte.  Returns the total."""
    import torch
    nat = gsp._native
    with_total = torch.full((n + 1,), -7, dtype=torch.int32, device="cuda")
    with_null = with_total.clone()
    total = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    nat.call(name, *args, with_total, total, nat.stream_ptr())
    nat.call(name, *args, with_null, None, nat.stream_ptr())
    nnz = int(total.item())
    assert nnz == int(with_total[-1].item()), name
    assert torch.equal(with_total, with_null), name
    return nnz


# ------------------------------------------------------------------------- matrices
def _random(n, density, seed, symmetric):
    rng = np.random.default_rng(seed)
    M = sparse.random(n, n, density, random_state=rng, format="csr")
    M.data = np.round(M.data * 4) - 1                     # stored zeros and negative values
    if symmetric:
        M = sparse.triu(M, 1)
        M = (M + M.T).tocsr()
    M.sort_indices()
    return M.astype(np.float32)


MATRICES = {
    "n0": lambda: sparse.csr_matrix((0, 0), dtype=np.float32),
    "n1": lambda: sparse.csr_matrix((1, 1), dtype=np.float32),
    "n1_loop": lambda: sparse.csr_matrix(np.ones((1, 1), np.float32)),
    "empty_rows": lambda: sparse.csr_matrix(
        ([1.0, 2.0, 0.0], [4, 0, 2], [0, 0, 1, 1, 3, 3]), shape=(5, 5), dtype=np.float32),
    "directed": lambda: _random(300, 0.03, 1, False),
    "undirected": lambda: _random(1000, 0.01, 2, True),
}


def _device(gsp, M, sfx):
    import torch
    dt = torch.float32 if sfx == "f32" else torch.float64
    return gsp.graphs.csr.DeviceCSR.from_scipy(M, dt, "cuda")


def _host_transpose(gsp, M, sfx):
    T = M.T.tocsr()
    T.sort_indices()
    return _device(gsp, T, sfx)


@pytest.mark.parametrize("sfx", SFX)
@pytest.mark.parametrize("name", sorted(MATRICES))
def test_matrix_counts(gsp, name, sfx):
    """Compaction, 'average', the four other symmetrisations, both Laplacians and the incidence
    matrix of each matrix of the zoo."""
    import torch
    nat = gsp._native
    M = MATRICES[name]()
    n = M.shape[0]
    A, B = _device(gsp, M, sfx), _host_transpose(gsp, M, sfx)
    assert counted(gsp, "gsp_csr_compact_count_" + sfx, n, nat.i64(n), A.indptr, A.data) == \
        np.count_nonzero(M.data)
    operands = (A.indptr, A.indices, A.data, B.indptr, B.indices, B.data)
    counted(gsp, "gsp_csr_average_count_" + sfx, n, nat.i64(n), *operands)
    for mode in range(4):
        counted(gsp, "gsp_csr_symmetrize_count_" + sfx, n, nat.i64(n), nat.i32(mode), *operands)
    dw = torch.from_numpy(np.asarray(abs(M).sum(axis=1), np.float64).ravel()).cuda()
    for lap_type in (0, 1):
        counted(gsp, "gsp_laplacian_count_" + sfx, n, nat.i64(n), A.indptr, A.indices, A.data,
                dw, nat.i32(lap_type))
    counted(gsp, "gsp_incidence_count", n, nat.i64(n), A.indptr, A.indices, None, None)
    if M.nnz:                                  # an empty W^T's indices are a NULL pointer
        counted(gsp, "gsp_incidence_count", n, nat.i64(n), A.indptr, A.indices, B.indptr,
                B.indices)


@pytest.mark.parametrize("name", sorted(MATRICES))
def test_subgraph_counts(gsp, name):
    """Induced submatrices with repeated vertices, with and without labels, and of no vertex."""
    import torch
    nat = gsp._native
    M = MATRICES[name]()
    n = M.shape[0]
    A = _device(gsp, M, "f32")
    rng = np.random.default_rng(n)
    labels = torch.from_numpy(rng.integers(0, 3, n).astype(np.int32)).cuda()
    for m in (0, 2 * n + 1 if n else 0):
        v = torch.from_numpy(rng.integers(0, max(n, 1), m).astype(np.int32)).cuda()
        mptr = torch.empty(n + 1, dtype=torch.int32, device="cuda")
        mpos = torch.empty(m, dtype=torch.int32, device="cuda")
        nat.call("gsp_vertex_map", nat.i64(n), nat.i64(m), v, mptr, mpos, nat.stream_ptr())
        for lab in (None, labels):
            counted(gsp, "gsp_subgraph_count", m, nat.i64(m), A.indptr, A.indices, v, mptr, lab)


def test_closed_form_counts(gsp):
    """Grid2d, the path / comet / star family, the torus, the complete graph and the random ring:
    the total is also the count the closed form gives."""
    import torch
    nat = gsp._native
    for n1, n2 in ((1, 1), (1, 5), (7, 3), (64, 129)):
        assert counted(gsp, "gsp_grid2d_count", n1 * n2, nat.i64(n1), nat.i64(n2)) == \
            2 * (n1 * (n2 - 1) + n2 * (n1 - 1))
    for n, k, directed in ((0, 0, 0), (1, 0, 0), (2, 0, 1), (9, 0, 1), (7, 3, 0), (40, 39, 0)):
        want = (n - 1 if directed else 2 * (n - 1)) if n else 0
        assert counted(gsp, "gsp_comet_count", n, nat.i64(n), nat.i64(k), nat.i32(directed)) == \
            want
    for nv, mv in ((1, 1), (2, 3), (5, 7)):              # sides of 1 and 2 merge neighbours
        counted(gsp, "gsp_torus_count", nv * mv, nat.i64(nv), nat.i64(mv))
    assert counted(gsp, "gsp_torus_count", 300 * 200, nat.i64(300), nat.i64(200)) == 4 * 60000
    for n in (0, 1, 2, 50):
        assert counted(gsp, "gsp_full_connected_indptr", n, nat.i64(n)) == n * (n - 1)
    drawn = np.sort(np.random.default_rng(0).uniform(0, 6.28, 1000))
    for angles in ([0.0, 1.0, 2.0], [0.0, 1.0, 1.0, 2.0], drawn):     # a zero gap is not stored
        a = torch.tensor(angles, dtype=torch.float64, device="cuda")
        zeros = int((np.diff(angles) == 0).sum())
        assert counted(gsp, "gsp_random_ring_count", len(angles), nat.i64(len(angles)), a) == \
            2 * (len(angles) - zeros)


def test_radius_counts(gsp):
    import torch
    nat = gsp._native
    rng = np.random.default_rng(3)
    for n, d, eps in ((1, 2, 1.0), (50, 2, 0.3), (700, 3, 0.2), (700, 5, 0.0)):
        pts = torch.from_numpy(rng.uniform(size=(n, d))).cuda()
        counted(gsp, "gsp_radius_count", n, nat.i64(n), nat.i32(d), pts, nat.f64(eps),
                nat.f64(2.0))


def test_line_graph_counts(gsp):
    """Undirected and directed graphs, with loops, and a graph without edges."""
    nat = gsp._native
    loops = sparse.identity(30, format="csr", dtype=np.float32) + _random(30, 0.2, 4, True)
    for W in (_random(1000, 0.01, 2, True), _random(300, 0.03, 1, False), loops,
              sparse.csr_matrix((6, 6), dtype=np.float32)):
        W.eliminate_zeros()
        W.data = np.abs(W.data)
        G = gsp.graphs.Graph(W)
        G.compute_differential_operator()
        _, s, t, _, _ = G._edges_device()
        ne = G.n_edges
        counted(gsp, "gsp_line_graph_count", ne, nat.i64(ne), s, t, G.D.indptr, G.W.indptr,
                G.W.indices, nat.i32(G.is_directed()))


# --------------------------------------------------------------- past 2^31 entries
def _need_free(nbytes):
    import torch
    if torch.cuda.mem_get_info()[0] < nbytes:
        pytest.skip("needs %d GB of free device memory" % (nbytes >> 30))


def test_grid2d_count_past_int32(gsp):
    """The count of Grid2d(33600, 33600) reports its 4 515 705 600 entries in int64, where the
    int32 scan has wrapped to a positive number of entries that a fill would overrun."""
    import torch
    nat = gsp._native
    _need_free(8 << 30)
    n = GRID * GRID
    indptr = torch.empty(n + 1, dtype=torch.int32, device="cuda")        # 4.5 GB
    total = torch.empty(1, dtype=torch.int64, device="cuda")
    nat.call("gsp_grid2d_count", nat.i64(GRID), nat.i64(GRID), indptr, total, nat.stream_ptr())
    assert int(total.item()) == GRID_NNZ == 4_515_705_600
    assert int(indptr[-1].item()) == GRID_NNZ % 2 ** 32 == 220_738_304
    del indptr, total
    torch.cuda.empty_cache()


def test_grid2d_refused_before_allocating(gsp):
    import torch
    _need_free(8 << 30)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    with pytest.raises(ValueError, match="%d entries" % GRID_NNZ):
        gsp.graphs.Grid2d(GRID, GRID)
    # indptr and the total, each rounded up to the allocator's 512-byte blocks
    assert torch.cuda.max_memory_allocated() - before <= 4 * (GRID * GRID + 1) + 512 + 512
    gc.collect()                  # the traceback's frames hold the 4.5 GB indptr
    torch.cuda.empty_cache()
