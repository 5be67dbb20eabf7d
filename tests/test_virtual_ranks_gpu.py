"""The vertex-partitioned operator with several ranks on ONE device, against the single-GPU engine.

A rank is a set of device buffers, a flag array and a plan, so P ranks can live in one process:
their peer stores are then plain global stores into each other's windows.  The partitioned call
(``gsp_cheby_op_dist_phases_*``) is run phase by phase -- phase j of every rank before phase j + 1
of any, all on the current stream -- and before every launch the host reads the rank's flag array
and requires that everything the phase waits for is already published.  So no launch ever waits
on something that is not yet in memory.  This runs the halo tiles of the fused step (wait,
coherent gathers, peer stores, publish counter), the front / interior split, the separate wait /
step / push kernels, the sequence numbers and buffer rotation and the peer tables of
``distributed.PeerTables``.  It does not test the protocol under real concurrency between ranks
(memory ordering of peer stores against flags, IPC mappings): that needs several GPUs
(tests/test_distributed_gpu.py).

After every phase, every rank's owned rows and halo rows of the block just written equal the
single-GPU block bit for bit, every flag slot holds exactly the published value, the push
counters are back to zero and rows no one may write still hold a NaN-payload sentinel.  At the
end the result equals ``cheby_op_device`` (forward form) or ``cheby_clenshaw_device`` (Clenshaw
form) on the whole graph bit for bit.  Each rank's step phases must also have taken the exchange
the case was built for: the fused step, or separate wait / step / push kernels (told apart by the
number of kernels launched).
"""
import ctypes
import time
import types

import numpy as np
import pytest
from scipy import sparse

from oracle import pygsp_oracle as orc
from oracle import step_oracle as so

pytestmark = pytest.mark.gpu

SENTINEL = {4: 0x7FE5A5A5, 8: 0x7FF5A5A5A5A5A5A5}     # quiet NaNs with a payload, by item size
N_BUFS = 3


@pytest.fixture(scope="module")
def torch():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch


def _launches():
    from pygsp_b200 import _native as nat
    fn = nat.lib().gsp_launch_count
    fn.restype = ctypes.c_uint64
    return int(fn())


def _int_view(torch, t):
    return t.view(torch.int32 if t.element_size() == 4 else torch.int64)


# ------------------------------------------------------------------------------------ graphs ---
def _laplacian(W, dtype):
    L = orc.laplacian(sparse.csr_matrix(W)).astype(dtype)
    L.sort_indices()
    return L


def _sensor(n, seed=3, k=8):
    return sparse.csr_matrix(so.sensor_adjacency(n, k=k, seed=seed))


def _grid(rows, cols):
    """Adjacency of a rows x cols grid, 4 neighbours, row-major numbering."""
    idx = np.arange(rows * cols).reshape(rows, cols)
    a = np.concatenate([idx[:, :-1].ravel(), idx[:-1, :].ravel()])
    b = np.concatenate([idx[:, 1:].ravel(), idx[1:, :].ravel()])
    W = sparse.csr_matrix((np.ones(2 * a.size), (np.r_[a, b], np.r_[b, a])),
                          shape=(rows * cols,) * 2)
    W.sort_indices()
    return W


def _exchange_from(L, bounds):
    """``exchange_ids`` answered from the global matrix: rank q asks owner r for the columns of
    its rows that r owns, ascending, as the all-to-all-v of ``_exchange_ids_torch`` delivers."""
    P = len(bounds) - 1
    halos = []
    for q in range(P):
        cols = L[bounds[q]:bounds[q + 1]].indices
        halos.append(np.unique(cols[(cols < bounds[q]) | (cols >= bounds[q + 1])]).astype(np.int64))

    def ex(halo_ids, recv_counts, rank, parts, group):
        lo, hi = bounds[rank], bounds[rank + 1]
        asked = [h[(h >= lo) & (h < hi)] if q != rank else h[:0] for q, h in enumerate(halos)]
        return np.concatenate(asked), np.array([a.size for a in asked], dtype=np.int64)
    return ex


# ------------------------------------------------------------------------------------- world ---
class World:
    """P ranks on the current device: per rank one allocation laid out like ``PeerWindow``'s
    (buf0 | buf1 | buf2 | flags[P] | counters), zeroed, halo and padding rows set to the
    sentinel, and its ``gsp_dist_plan`` from ``distributed.PeerTables``."""

    def __init__(self, torch, L, bounds, dtype, nsig, nscales, plans=None, separate=False):
        from pygsp_b200 import distributed as gd
        from pygsp_b200 import _native as nat
        self.torch, self.nat = torch, nat
        self.bounds = np.asarray(bounds, dtype=np.int64)
        self.P = P = len(bounds) - 1
        self.dtype, self.nsig, self.nscales = dtype, nsig, nscales
        ex = _exchange_from(L, self.bounds)
        self.plans = plans or [gd.HaloPlan(L[bounds[r]:bounds[r + 1]], self.bounds, r,
                                           exchange_ids=ex) for r in range(P)]
        dev = torch.device("cuda")
        self.item = item = torch.empty((), dtype=dtype).element_size()
        self.mem, self.bufs, self.flags, self.counters, self.bb = [], [], [], [], []
        for p in self.plans:
            ext = p.n_local + p.n_halo
            bb = ((ext * nsig * item + 255) // 256) * 256
            foff = N_BUFS * bb
            mem = torch.zeros(foff + 8 * P + 256, dtype=torch.uint8, device=dev)
            _int_view(torch, mem[:foff].view(dtype)).fill_(SENTINEL[item])
            bufs = [mem[b * bb:b * bb + ext * nsig * item].view(dtype).view(ext, nsig)
                    for b in range(N_BUFS)]
            for b in bufs:
                b[:p.n_local].zero_()
            self.mem.append(mem)
            self.bb.append(bb)
            self.bufs.append(bufs)
            self.flags.append(mem[foff:foff + 8 * P].view(torch.int64))
            self.counters.append(mem[foff + 8 * P:foff + 8 * P + 16].view(torch.int64))
        infos = [(p.n_local, p.recv_counts.tolist(), bb) for p, bb in zip(self.plans, self.bb)]
        bases = [m.data_ptr() for m in self.mem]
        t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(device=dev, dtype=dt)
        self.csr, self.tables, self.tiles, self.perm, self.halo = [], [], [], [], []
        for p in self.plans:
            csr = (t(p.indptr, torch.int32), t(p.indices, torch.int32), t(p.data, dtype))
            tab = gd.PeerTables(p, infos, bases, *csr, t(p.send_idx, torch.int64), N_BUFS)
            tab.dist_plan.separate_exchange = int(separate)
            tile = None
            if dtype == torch.float32:
                tile = nat.TilePlan()
                nat.call("gsp_cheby_tile_plan", nat.i64(p.n_local), csr[0], nat.i64(nsig),
                         nat.i32(nscales), tile, nat.stream_ptr())
                tile = tile if tile.rows_per_tile > 0 else None
            self.csr.append(csr)
            self.tables.append(tab)
            self.tiles.append(tile)
            self.perm.append(t(p.perm, torch.int64))
            self.halo.append(t(p.halo_ids, torch.int64))
        self.neighbors = [tab.neighbors for tab in self.tables]
        self.pushed = [set() for _ in range(P)]     # blocks whose halo rows a neighbour wrote
        self.seq = 0
        self.record = {}                             # (call, rank, phase) -> kernels launched

    # ------------------------------------------------------------------- which exchange ---
    def fusable(self, r):
        p, tab, tile = self.plans[r], self.tables[r], self.tiles[r]
        if tile is None or tab.dist_plan.separate_exchange or not 1 <= len(tab.neighbors) <= 32:
            return False
        R = tile.rows_per_tile
        return max(tab.n_push_rows, p.n_true_boundary) <= (p.n_local // R) * R

    def step_launches(self, r, path, publish):
        """Kernels one recurrence step of rank r launches on the given exchange path."""
        p, tab, tile = self.plans[r], self.tables[r], self.tiles[r]
        n = p.n_local
        if tile is None:
            steps, full, rem = int(n > 0), 0, 0
        else:
            R = tile.rows_per_tile
            full, rem = (n // R) * R, n % R
            steps = int(full > 0) + int(rem > 0)
        if path == "fused":
            R = tile.rows_per_tile
            front = -(-max(tab.n_push_rows if publish else 0, p.n_true_boundary) // R) * R
            return int(front > 0) + int(full - front > 0) + int(rem > 0)
        return int(len(tab.neighbors) > 0) + steps + int(publish)

    # ------------------------------------------------------------------------- one call ---
    def call(self, lmax, c, xs, clenshaw, use_perm, check=None):
        """Runs one call of every rank phase by phase; ``check(phase, base)`` after each phase.
        xs[r]: rank r's input (caller's order with ``use_perm``, else local order)."""
        torch, nat = self.torch, self.nat
        nscales, m = c.shape
        K = m - 1
        base = self.seq
        seqs = [ctypes.c_uint64(base) for _ in range(self.P)]
        rs = [torch.empty((nscales, p.n_local, self.nsig), dtype=self.dtype, device="cuda")
              for p in self.plans]
        call_id = base // (m + 2)
        for r in range(self.P):
            self.tables[r].dist_plan.perm = self.perm[r].data_ptr() if use_perm else None
        for phase in range(K + 2):
            for r in range(self.P):
                # the safety rule: everything this phase waits for is already in memory
                torch.cuda.synchronize()
                if phase >= 1:
                    seen = self.flags[r].cpu().numpy()
                    for q in self.neighbors[r]:
                        assert seen[q] >= base + phase, (r, phase, q, seen[q], base)
                before = _launches()
                nat.call("gsp_cheby_op_dist_phases_" + nat.suffix(self.dtype),
                         self.tables[r].dist_plan, self.tiles[r], nat.f64(lmax), c,
                         nat.i32(nscales), nat.i32(m), xs[r], nat.i64(self.nsig), rs[r],
                         nat.i32(int(clenshaw)), ctypes.byref(seqs[r]), nat.i32(phase),
                         nat.i32(phase + 1), nat.stream_ptr())
                self.record[(call_id, r, phase)] = _launches() - before
                assert seqs[r].value == (base + m + 2 if phase == K + 1 else base)
            torch.cuda.synchronize()
            if check is not None:
                check(phase, base)
        self.seq = base + m + 2
        return rs


def _written(phase, K, clenshaw):
    """(buffer the phase writes, whether its boundary rows are pushed); None: the caller's r."""
    if phase == 1:
        return 0, True
    s = phase - 1
    if not clenshaw:
        return s & 1, s < K
    if s == K:
        return None, False
    return (1 if s == 1 or s % 2 == 1 else 2), True


def _reference_blocks(torch, L, dtype, nsig, nscales, lmax, c, x, clenshaw):
    """The block each phase writes, from the single-GPU engine's step schedule: the same call
    on one rank that owns the whole graph (no halo, global row order)."""
    n = L.shape[0]
    ref = World(torch, L, [0, n], dtype, nsig, nscales)
    K = c.shape[1] - 1
    blocks = {}

    def snap(phase, base):
        b, _ = _written(phase, K, clenshaw)
        if phase >= 1 and b is not None:
            blocks[phase] = _int_view(torch, ref.bufs[0][b][:n].clone())
    r = ref.call(lmax, c, [x], clenshaw, False, snap)
    return blocks, r[0]


def run_case(torch, L, bounds, dtype, nsig, nscales, m, clenshaw, expect, separate=False,
             plans=None, seed=0):
    """One world, two calls; every check of the module docstring.  ``expect[r]``: 'fused' or
    'separate', the exchange rank r's steps must take.  Returns the world."""
    import pygsp_b200 as gsp
    from pygsp_b200.filters import approximations as apx
    t0 = time.perf_counter()
    n = L.shape[0]
    bounds = np.asarray(bounds, dtype=np.int64)
    rng = np.random.default_rng(seed)
    c = np.ascontiguousarray(rng.standard_normal((nscales, m)) / np.arange(1, m + 1))
    lmax = 1.01 * float(abs(L.astype(np.float64)).sum(axis=1).max())
    npdt = np.float32 if dtype == torch.float32 else np.float64
    x = torch.from_numpy(so.scaled_signals(rng, n, nsig, npdt)).cuda()
    K = m - 1
    cl = bool(clenshaw) and nscales == 1 and K >= 2
    blocks, _ = _reference_blocks(torch, L, dtype, nsig, nscales, lmax, c, x, cl)
    w = World(torch, L, bounds, dtype, nsig, nscales, plans=plans, separate=separate)
    assert [("fused" if w.fusable(r) else "separate") for r in range(w.P)] == list(expect)
    # forward form: input and result in local order; Clenshaw form: the caller's order (perm)
    lo = [int(b) for b in bounds[:-1]]
    if cl:
        xs = [x[lo[r]:lo[r] + p.n_local].contiguous() for r, p in enumerate(w.plans)]
    else:
        xs = [x[lo[r] + w.perm[r]].contiguous() for r in range(w.P)]
    sent = SENTINEL[w.item]

    def check(phase, base):
        value = base + 1 + min(phase, K)
        for r, p in enumerate(w.plans):
            expect_flags = np.zeros(w.P, dtype=np.int64)
            for q in w.neighbors[r]:
                expect_flags[q] = value
            np.testing.assert_array_equal(w.flags[r].cpu().numpy(), expect_flags,
                                          err_msg="flags of rank %d, phase %d" % (r, phase))
            ctr = w.counters[r].cpu().numpy()
            assert ctr[0] & 0xFFFFFFFF == 0 and ctr[1] == 0, (r, phase, ctr)
        if phase == 0:
            return
        b, pushed = _written(phase, K, cl)
        for r, p in enumerate(w.plans):
            if b is not None:
                got = _int_view(torch, w.bufs[r][b])
                ref = blocks[phase]
                assert torch.equal(got[:p.n_local], ref[lo[r] + w.perm[r]]), \
                    "owned rows of rank %d, phase %d" % (r, phase)
                if pushed and p.n_halo:
                    w.pushed[r].add(b)
                    assert torch.equal(got[p.n_local:], ref[w.halo[r]]), \
                        "halo rows of rank %d, phase %d" % (r, phase)
            for bi in range(N_BUFS):
                words = _int_view(torch, w.mem[r][bi * w.bb[r]:(bi + 1) * w.bb[r]].view(dtype))
                ext = (p.n_local + p.n_halo) * nsig
                assert bool((words[ext:] == sent).all()), "padding of rank %d" % r
                if bi not in w.pushed[r]:
                    assert bool((words[p.n_local * nsig:ext] == sent).all()), \
                        "halo rows of block %d of rank %d, phase %d" % (bi, r, phase)

    outs = []
    for _ in range(2):
        rs = w.call(lmax, c, xs, cl, cl, check)
        torch.cuda.synchronize()
        if cl:
            outs.append(torch.cat([r_[0] for r_ in rs]))
        else:
            out = torch.empty((nscales, n, nsig), dtype=dtype, device="cuda")
            for r in range(w.P):
                out[:, lo[r] + w.perm[r]] = rs[r]
            outs.append(out)
    assert torch.equal(_int_view(torch, outs[1]), _int_view(torch, outs[0])), "second call"
    dev = gsp.graphs.DeviceCSR.from_scipy(L, dtype, torch.device("cuda"))
    if cl:
        ref = apx.cheby_clenshaw_device(dev, lmax, c, x)
    else:
        ref = apx.cheby_op_device(dev, lmax, c, x)
    assert torch.equal(_int_view(torch, outs[0]), _int_view(torch, ref)), "single-GPU result"
    # a few columns against the float64 oracle
    cols = [0, nsig // 2, nsig - 1]
    want = orc.cheby_op(L.astype(np.float64), lmax, c, x[:, cols].double().cpu().numpy())
    got = outs[0].reshape(-1, nsig)[:, cols].double().cpu().numpy()
    err = np.abs(got - want).max(axis=0) / np.maximum(np.abs(want).max(axis=0), 1e-300)
    assert err.max() <= (1e-5 if dtype == torch.float32 else 1e-10), err
    # every step phase took the exchange the case was built for
    for (call_id, r, phase), got_n in w.record.items():
        if phase < 2:
            continue
        publish = phase - 1 < K
        assert got_n == w.step_launches(r, expect[r], publish), (call_id, r, phase, got_n)
        if w.neighbors[r] and expect[r] == "fused" and publish:
            assert w.step_launches(r, "separate", publish) != got_n
    print("\n[virtual ranks] P=%d %s nsig=%d nscales=%d m=%d %s paths=%s %.2fs"
          % (w.P, str(dtype)[6:], nsig, nscales, m, "clenshaw" if cl else "forward",
             "".join("F" if e == "fused" else "S" for e in expect), time.perf_counter() - t0))
    return w


# ------------------------------------------------------------------------------------- cases ---
SENSOR_N = 20000


@pytest.fixture(scope="module")
def sensor32():
    return _laplacian(_sensor(SENSOR_N), np.float32)


@pytest.mark.parametrize("P,nsig,nscales,m,clenshaw", [
    (2, 64, 1, 16, True), (2, 128, 1, 16, False), (2, 32, 16, 2, False),
    (3, 8, 2, 3, False), (3, 32, 1, 3, True), (3, 16, 1, 4, True),
    (4, 16, 3, 4, False), (4, 128, 1, 4, True), (4, 64, 2, 16, False), (4, 8, 1, 16, True),
])
def test_morton_sensor_even_bounds(torch, sensor32, P, nsig, nscales, m, clenshaw):
    """Thin halos of a Morton-ordered k-NN graph: every rank fuses its exchange."""
    from pygsp_b200 import distributed as gd
    run_case(torch, sensor32, gd.even_bounds(SENSOR_N, P), torch.float32, nsig, nscales, m,
             clenshaw, ["fused"] * P)


@pytest.mark.parametrize("dw", [-1, 0, 1])
@pytest.mark.parametrize("clenshaw", [False, True])
def test_grid_strips_around_one_tile(torch, dw, clenshaw):
    """Row strips of a grid of width R - 1, R and R + 1: the end ranks have `width` boundary
    rows, the middle rank 2 * width, so the counts are R - 1, R, R + 1 and cover every residue
    of the multiple-of-4 padding of HaloPlan (63, 64, 65, 126, 128, 130 for R = 64)."""
    probe = World(torch, _laplacian(_grid(8, 64), np.float32), [0, 512], torch.float32, 64, 1)
    R = probe.tiles[0].rows_per_tile
    width, height = R + dw, 40
    L = _laplacian(_grid(3 * height, width), np.float32)
    bounds = [0, height * width, 2 * height * width, 3 * height * width]
    w = run_case(torch, L, bounds, torch.float32, 64, 1, 5, clenshaw, ["fused"] * 3)
    assert [p.n_true_boundary for p in w.plans] == [width, 2 * width, width]


@pytest.mark.parametrize("clenshaw", [False, True])
def test_rank_smaller_than_a_tile_takes_the_separate_exchange(torch, sensor32, clenshaw):
    """One rank with fewer rows than a tile next to ranks that fuse, in the same world."""
    w = run_case(torch, sensor32, [0, 40, 10000, SENSOR_N], torch.float32, 64, 1, 6, clenshaw,
                 ["separate", "fused", "fused"])
    assert w.tiles[0] is None or w.plans[0].n_local < w.tiles[0].rows_per_tile


@pytest.mark.parametrize("extra,expect", [(0, ["fused"] * 2), (37, ["separate"] * 2)])
def test_renumbered_graph_every_row_a_boundary_row(torch, extra, expect):
    """A randomly renumbered k-NN graph: nearly every row reads the halo.  With blocks of whole
    tiles the front launch is the whole block and the interior launch is empty; with 37 more
    rows the boundary rows do not fit the full tiles and the exchange is separate."""
    n = 2 * 64 * 24 + 2 * extra
    W = _sensor(n, seed=9)
    p = np.random.default_rng(5).permutation(n)
    L = _laplacian(W[p][:, p], np.float32)
    w = run_case(torch, L, [0, n // 2, n], torch.float32, 64, 1, 5, True, expect)
    for r, pl in enumerate(w.plans):
        assert pl.n_true_boundary > 0.9 * pl.n_local
        if extra == 0:
            assert w.step_launches(r, "fused", True) == 1     # front only: no interior launch


def test_one_way_edges_push_more_rows_than_wait(torch, sensor32):
    """Entries L[i, j] with i in rank 1 and j an interior row of rank 0 (no entry L[j, i]): rank 0
    pushes rows that are not boundary rows, so n_push_rows > n_boundary_rows and the front launch
    has more push tiles than wait tiles."""
    from pygsp_b200 import distributed as gd
    bounds = gd.even_bounds(SENSOR_N, 2)
    ex = _exchange_from(sensor32, bounds)
    p0 = gd.HaloPlan(sensor32[:bounds[1]], bounds, 0, exchange_ids=ex)
    targets = p0.perm[p0.n_boundary:p0.n_boundary + 150]          # rank 0's first interior rows
    src = np.arange(bounds[1] + 3000, bounds[1] + 3000 + 150)     # inside rank 1's block
    one_way = sparse.csr_matrix((np.full(150, -0.25, np.float32), (src, targets)),
                                shape=sensor32.shape)
    L = (sensor32 + one_way).tocsr()
    L.sort_indices()
    w = run_case(torch, L, bounds, torch.float32, 32, 1, 7, True, ["fused", "fused"])
    R = w.tiles[0].rows_per_tile
    assert w.tables[0].n_push_rows > w.plans[0].n_true_boundary
    assert -(-w.tables[0].n_push_rows // R) > -(-w.plans[0].n_true_boundary // R)


def test_rank_without_neighbours(torch):
    """A disconnected block (rank 2) next to two ranks that exchange halos."""
    L = _laplacian(sparse.block_diag([_sensor(12000, seed=4), _sensor(6000, seed=6)]).tocsr(),
                   np.float32)
    w = run_case(torch, L, [0, 6000, 12000, 18000], torch.float32, 64, 2, 6, False,
                 ["fused", "fused", "separate"])
    assert w.neighbors[2] == [] and w.neighbors[0] == [1]


def test_hub_rank_with_33_neighbours(torch):
    """A hub vertex (in rank 0) joined to one vertex of every other block, P = 34: the hub's rank
    has 33 neighbours and takes the separate exchange; the others fuse."""
    P, per = 34, 900
    n = P * per
    W = _sensor(n, seed=8).tolil()
    for q in range(1, P):
        v = q * per + per // 2
        W[0, v] = W[v, 0] = 0.5
    L = _laplacian(W.tocsr(), np.float32)
    w = run_case(torch, L, np.arange(P + 1) * per, torch.float32, 16, 1, 4, True,
                 ["separate"] + ["fused"] * (P - 1))
    assert len(w.neighbors[0]) == 33


@pytest.mark.parametrize("clenshaw", [False, True])
def test_no_tile_plan_row_group_kernel(torch, sensor32, clenshaw):
    """nsig = 24 has no tile plan: every rank runs the row-group kernel and the separate
    exchange."""
    from pygsp_b200 import distributed as gd
    w = run_case(torch, sensor32, gd.even_bounds(SENSOR_N, 3), torch.float32, 24, 1, 5,
                 clenshaw, ["separate"] * 3)
    assert all(t is None for t in w.tiles)


@pytest.mark.parametrize("clenshaw", [False, True])
def test_float64_separate_exchange(torch, clenshaw):
    from pygsp_b200 import distributed as gd
    L = _laplacian(_sensor(SENSOR_N), np.float64)
    run_case(torch, L, gd.even_bounds(SENSOR_N, 3), torch.float64, 16, 2 - int(clenshaw), 6,
             clenshaw, ["separate"] * 3)


@pytest.mark.parametrize("clenshaw", [False, True])
def test_float32_forced_separate_exchange(torch, sensor32, clenshaw):
    from pygsp_b200 import distributed as gd
    run_case(torch, sensor32, gd.even_bounds(SENSOR_N, 2), torch.float32, 64, 1, 8, clenshaw,
             ["separate"] * 2, separate=True)


# ------------------------------------------------------------------------------- one rank ---
def _permuted_plan(L, perm):
    """A one-rank plan whose local order is the random permutation ``perm``: row i of the local
    CSR is row perm[i] of L, columns renamed to match, entries in the same order."""
    n = L.shape[0]
    inv = np.empty(n, dtype=np.int64)
    inv[perm] = np.arange(n)
    Lp = L[perm].tocsr()                           # row order changes, within-row order kept
    return types.SimpleNamespace(
        rank=0, parts=1, bounds=np.array([0, n]), n_local=n, n_global=n, n_halo=0,
        halo_ids=np.zeros(0, np.int64), recv_counts=np.zeros(1, np.int64),
        send_counts=np.zeros(1, np.int64), send_idx=np.zeros(0, np.int64), perm=perm,
        inv_perm=inv, n_boundary=0, n_true_boundary=0, indptr=Lp.indptr.astype(np.int32),
        indices=inv[Lp.indices].astype(np.int32), data=Lp.data, nnz=Lp.nnz)


@pytest.mark.parametrize("clenshaw", [False, True])
def test_one_rank_phased_whole_and_permuted(torch, sensor32, clenshaw):
    """One rank: the phased call gives the bits of the whole call, and a whole call with a random
    row permutation (the local CSR renumbered to match) gives the unpermuted call's bits in the
    caller's order -- the forward form's gather and scatter of rows, and the Clenshaw form's
    gather and permuted last store.  A phased forward call refuses the permutation before any
    launch."""
    from pygsp_b200 import _native as nat
    L = sensor32
    n, nsig, nscales, m = L.shape[0], 64, 1 if clenshaw else 3, 9
    rng = np.random.default_rng(7)
    c = np.ascontiguousarray(rng.standard_normal((nscales, m)) / np.arange(1, m + 1))
    lmax = 1.01 * float(abs(L.astype(np.float64)).sum(axis=1).max())
    x = torch.from_numpy(so.scaled_signals(rng, n, nsig)).cuda()

    def whole(w, use_perm):
        d = w.tables[0].dist_plan
        d.perm = w.perm[0].data_ptr() if use_perm else None
        r = torch.empty((nscales, n, nsig), dtype=torch.float32, device="cuda")
        seq = ctypes.c_uint64(w.seq)
        nat.call("gsp_cheby_op_dist_f32", d, w.tiles[0], nat.f64(lmax), c, nat.i32(nscales), nat.i32(m), x,
                 nat.i64(nsig), r, nat.i32(int(clenshaw)), ctypes.byref(seq), nat.stream_ptr())
        assert seq.value == w.seq + m + 2
        w.seq = seq.value
        torch.cuda.synchronize()
        return r

    plain = World(torch, L, [0, n], torch.float32, nsig, nscales)
    a = whole(plain, False)
    b = plain.call(lmax, c, [x], clenshaw, False)[0]
    torch.cuda.synchronize()
    assert torch.equal(_int_view(torch, b), _int_view(torch, a))
    perm = np.random.default_rng(8).permutation(n).astype(np.int64)
    pw = World(torch, L, [0, n], torch.float32, nsig, nscales, plans=[_permuted_plan(L, perm)])
    assert torch.equal(_int_view(torch, whole(pw, True)), _int_view(torch, a))
    if not clenshaw:
        d = pw.tables[0].dist_plan
        d.perm = pw.perm[0].data_ptr()
        seq = ctypes.c_uint64(pw.seq)
        before = _launches()
        r = torch.empty((nscales, n, nsig), dtype=torch.float32, device="cuda")
        assert pw.neighbors[0] == []          # the flag check: a single rank waits for nobody
        with pytest.raises(nat.NativeError, match="phased forward call takes no row permutation"):
            nat.call("gsp_cheby_op_dist_phases_f32", d, pw.tiles[0], nat.f64(lmax), c,
                     nat.i32(nscales), nat.i32(m), x, nat.i64(nsig), r, nat.i32(0),
                     ctypes.byref(seq), nat.i32(0), nat.i32(m), nat.stream_ptr())
        assert _launches() == before and seq.value == pw.seq
