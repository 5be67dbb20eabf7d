/* libgspb200 -- C ABI of the H100-native Chebyshev graph-filtering engine.
 *
 * The reference (PyGSP 0.6.1) has no FFI: its seam for this path is the Python
 * call boundary, below which every operation is a call into SciPy's compiled
 * sparsetools / ARPACK.  Each entry point below replaces one such call; the
 * comment names the reference line it stands in for.  Conventions:
 *
 *   - every array argument is a DEVICE pointer unless its name ends in _host;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it and
 *     nothing synchronises (the caller owns synchronisation);
 *   - return value 0 = OK, negative = error (-1 bad argument, -2 CUDA error,
 *     -3 unsupported); the message is available from gsp_last_error()
 *     (thread-local).  Nothing throws across the boundary;
 *   - the callee never frees or keeps caller memory.  A CSR output whose size
 *     is data dependent comes as a *_count / *_fill pair.  The count writes
 *     the output indptr and, through its `int64_t* nnz` argument (device, may
 *     be NULL), the number of entries as an int64; indptr is meaningful only
 *     when *nnz < 2^31, which the caller checks before it allocates the fill's
 *     outputs;
 *   - CSR index arrays are int32 (as SciPy's for nnz < 2^31), values are
 *     float (_f32) or double (_f64); the weighted degree `dw` is always double.
 */
#ifndef GSPB200_H_
#define GSPB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSPB200_ABI_VERSION 3

int gsp_abi_version(void);
const char* gsp_last_error(void);
/* number of kernels this library has launched since it was loaded */
uint64_t gsp_launch_count(void);
int gsp_device_info(int* sm_count, int* cc_major, int* cc_minor, int64_t* l2_bytes);

/* ------------------------------------------------------------------ filter --
 * gsp_cheby_op_*: pygsp/filters/approximations.py:58-114 `cheby_op(G, c, signal)`.
 *   L = (indptr, indices, data) n x n CSR; lmax = G.lmax; coeffs_host is the
 *   (nscales, m) row-major coefficient matrix (m = order + 1 >= 2, else the
 *   reference's TypeError condition is reported as -1); x is (n, nsig)
 *   row-major; r receives (nscales, n, nsig) = the reference's filter-major
 *   (nscales*n, nsig) block; work holds 2*n*nsig elements.  x is not modified.
 *   nnz = number of stored entries of L; plan_host may be NULL (row-group kernel).
 * gsp_cheby_step_*: one fused recurrence step on rows [row_begin, row_end)
 *   x_new = alpha*(L x_cur) + beta*x_cur + gamma*x_old ;  r_i (+)= ck[i]*x_new
 *   (first != 0: r_i = c0[i]/2 * x_cur + ck[i] * x_new, x_old unused).
 *   x_new may alias x_old.  Stands for approximations.py:99-103 (first) and
 *   :107-112 (k >= 2).  Used directly by the vertex-partitioned multi-GPU path,
 *   where column indices address a local x_cur that has halo rows appended.
 * gsp_cheby_clenshaw_*: out = sum_i p_i(L) s_i for nsrc source blocks s_i ((nsrc, n, nsig) in
 *   memory) and coefficient rows c_i ((nsrc, m) row-major), by ONE backward (Clenshaw)
 *   recurrence on an (n, nsig) block: K SpMMs in total and no accumulator.  nsrc = 1 is the
 *   single-filter evaluation; nsrc = Nf is the synthesis of filter.py:313-322 (which runs Nf
 *   forward recurrences).  out is (n, nsig), work 2*n*nsig.  Same value as the forward
 *   recurrence, different rounding.
 * gsp_spmm_*: y = L x, scipy `csr_matrix.dot` (approximations.py:99, graph.py:955).  n is the
 *   number of ROWS of the matrix; x is read at the column indices only, so the matrix may be
 *   rectangular (n x m with x of m rows), as the differential operator's D and D^T are
 *   (difference.py:244, 331).  gsp_spmv_* below is for square matrices only (its window form
 *   stages x at the rows of its own tile).
 */
/* Tiling of the float32 fast path (TMA-staged row tiles, csrc/cheby_tiled.cu).
 * Filled by gsp_cheby_tile_plan() once per (matrix, nsig, nscales); all zeros
 * means "use the row-group kernel".  Plain host struct, owned by the caller. */
typedef struct gsp_tile_plan {
  int rows_per_tile;   /* rows of L per shared-memory stage */
  int slab_capacity;   /* CSR entries a stage can hold (>= the matrix's largest tile) */
  int stages;          /* depth of the TMA ring of steps that stage vector tiles (a step whose
                          stage holds only the CSR slab -- the first step, or x_old / r read
                          directly as in the Clenshaw form -- runs a one-stage ring) */
  int consumer_warps;  /* warps that compute (one more warp produces); the two-packet lane
                          mapping of the Clenshaw form runs min(consumer_warps, 8) of them */
  int gather_unroll;   /* reserved (always 4: one LDS.128 group of CSR entries) */
  int blocks_per_sm;   /* 0 = as many as fit */
} gsp_tile_plan;

/* Reads the matrix's largest tile (synchronises `stream` once) and chooses the tiling. */
int gsp_cheby_tile_plan(int64_t n, const int32_t* indptr, int64_t nsig, int nscales,
                        gsp_tile_plan* plan_host_out, void* stream);

/* Halo exchange fused into the tiled float32 step (vertex-partitioned path).  Local rows
 * are ordered boundary-first: rows [0, n_boundary_rows) may reference halo columns
 * (column ids >= n_owned), rows [0, n_push_rows) are needed by some neighbour.  A step is two
 * launches on the caller's stream.  First the tiles that hold such rows ("front" tiles, a few
 * dozen): their warps wait until flags[wait_ids[q]] >= wait_value (the neighbours have stored
 * x_cur's halo rows into this GPU; front tiles gather through L2, never through the
 * non-coherent path), every row < n_push_rows of x_new is stored into
 * peer_base[push_peer[e]][push_row[e], :] for e in [push_ptr[row], push_ptr[row+1]) (peer
 * stores over NVLink) and, with publish != 0, publish_value is written to every
 * peer_flags[q] when the last front tile is done -- at that point the pushed rows are visible
 * and nobody on this GPU reads the halo of x_cur any more, so the neighbours may also
 * overwrite it.  Then all interior tiles, with the plain kernel instantiation (one kernel
 * for both spills registers into the interior loop and runs slower).  All pointers are
 * device pointers; the struct itself is a host struct.  n_push_tiles / n_wait_tiles are
 * filled in by the library. */
typedef struct gsp_halo_fusion {
  int64_t n_push_rows;
  int64_t n_push_tiles;
  const int32_t* push_ptr;
  const int32_t* push_peer;
  const int64_t* push_row;
  void* const* peer_base;          /* float* const*  : peers' x_new buffers */
  uint64_t* const* peer_flags;     /* my slot in each neighbour's flag array */
  uint64_t* push_counter;          /* one zero-initialised device uint64 */
  const uint64_t* wait_flags;      /* my own flag array */
  const int32_t* wait_ids;         /* neighbour ranks to wait for */
  uint64_t publish_value;
  uint64_t wait_value;
  int32_t n_neighbors;
  int32_t n_wait;
  int64_t n_boundary_rows;         /* rows [0, n_boundary_rows) may read halo columns */
  int64_t n_wait_tiles;
  int64_t n_owned;                 /* columns >= n_owned are halo rows of x_cur */
  int32_t publish;                 /* 0: last step of a call, nothing is published */
  int32_t reserved;
} gsp_halo_fusion;

/* One fused step on the whole local row block with the halo exchange folded in
 * (float32, tiled kernel required: returns -3 when no tile plan applies).  reverse != 0
 * walks the interior tiles from the last to the first (alternate it between steps: the
 * lines a step wrote last are then the first ones the next step reads, still in L2). */
int gsp_cheby_step_halo_f32(int first, int64_t n_rows, int64_t nnz, const int32_t* indptr,
                            const int32_t* indices, const float* data, const float* x_cur,
                            const float* x_old, float* x_new, float* r, int64_t r_rows,
                            int64_t nsig, int nscales, const double* ck_host,
                            const double* c0_host, double alpha, double beta, double gamma,
                            int reverse, const gsp_tile_plan* plan_host,
                            const gsp_halo_fusion* halo_host, void* stream);

#define GSPB200_DECLARE_CHEBY_API(SUF, T)                                                         \
  int gsp_cheby_op_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,   \
                         const T* data, double lmax, const double* coeffs_host, int nscales,      \
                         int m, const T* x, int64_t nsig, T* r, T* work,                          \
                         const gsp_tile_plan* plan_host, void* stream);                           \
  int gsp_cheby_step_##SUF(int first, int64_t row_begin, int64_t row_end, int64_t nnz,            \
                           const int32_t* indptr, const int32_t* indices, const T* data,          \
                           const T* x_cur, const T* x_old, T* x_new, T* r, int64_t r_rows,        \
                           int64_t nsig, int nscales, const double* ck_host,                      \
                           const double* c0_host, double alpha, double beta, double gamma,        \
                           const gsp_tile_plan* plan_host, void* stream);                         \
  int gsp_cheby_clenshaw_##SUF(int64_t n, int64_t nnz, const int32_t* indptr,                     \
                               const int32_t* indices, const T* data, double lmax,                \
                               const double* coeffs_host, int nsrc, int m, const T* sources,      \
                               int64_t nsig, T* out, T* work, const gsp_tile_plan* plan_host,     \
                               void* stream);                                                     \
  int gsp_spmm_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices, const T* data,     \
                     const T* x, int64_t nsig, T* y, void* stream);

GSPB200_DECLARE_CHEBY_API(f32, float)
GSPB200_DECLARE_CHEBY_API(f64, double)

/* Filter banks wider than 16 filters (csrc/cheby_bank.cu).
 *
 * gsp_cheby_op_basis_*: pygsp/filters/approximations.py:58-114 `cheby_op(G, c, signal)` for any
 *   number of filters.  The m - 1 recurrence steps write T_k x into slot k of basis
 *   ((m, n, nsig), caller-given; slot 0 stands for T_0 = x and is read only when x is slot 0
 *   itself, otherwise it is not written), with no accumulator; then one combine pass forms
 *   r_i = sum_k c_ik T_k x for every filter, reading the basis once and writing each output once.
 *   coeffs is a DEVICE (nscales, m) row-major double matrix; r receives (nscales, n, ldr) with
 *   ldr >= nsig (a column range of a wider block: row j of filter i at r + (i n + j) ldr).  The
 *   combine forms fma(c_i1, T_1, (c_i0/2) T_0), then fma(c_ik, T_k, r) for increasing k, with the
 *   coefficients cast to T as the fused step casts them, so r is the bits of gsp_cheby_op_* on
 *   the same block.  Every step is one gsp_cheby_step_* (plan_host: the tiling for nscales = 0).
 *   No allocation, no synchronisation.
 * gsp_cheby_synthesis_wide_*: filter.py:313-322 (the synthesis of an Nf-feature signal, one
 *   forward recurrence per feature) for any nsrc.  One mix pass over the nsrc source blocks
 *   ((nsrc, n, nsig) in memory) forms the per-order sources u_k = sum_f c'_fk s_f (c'_f0 =
 *   c_f0 / 2, the sum in increasing f) for up to 32 orders, one more pass per further 32; then
 *   one Clenshaw recurrence b_k = u_k + 2 Lt b_{k+1} - b_{k+2} runs with the source block of
 *   order k (m - 1 SpMMs).  coeffs is a DEVICE (nsrc, m) row-major double matrix; out is
 *   (n, nsig); work holds (m + 2) n nsig elements; plan_host is the tiling for nscales = 1.
 *   Same value as gsp_cheby_clenshaw_*, different rounding (the sources are summed per order
 *   before they enter the recurrence).  No allocation, no synchronisation. */
#define GSPB200_DECLARE_BANK_API(SUF, T)                                                          \
  int gsp_cheby_op_basis_##SUF(int64_t n, int64_t nnz, const int32_t* indptr,                     \
                               const int32_t* indices, const T* data, double lmax,                \
                               const double* coeffs, int nscales, int m, const T* x,              \
                               int64_t nsig, T* basis, T* r, int64_t ldr,                         \
                               const gsp_tile_plan* plan_host, void* stream);                     \
  int gsp_cheby_synthesis_wide_##SUF(int64_t n, int64_t nnz, const int32_t* indptr,               \
                                     const int32_t* indices, const T* data, double lmax,          \
                                     const double* coeffs, int nsrc, int m, const T* sources,     \
                                     int64_t nsig, T* out, T* work,                               \
                                     const gsp_tile_plan* plan_host, void* stream);

GSPB200_DECLARE_BANK_API(f32, float)
GSPB200_DECLARE_BANK_API(f64, double)

/* Clenshaw filtering of ONE float32 source with the middle steps run two per launch.  A paired
 * launch forms b_k into a third work block and b_{k-1} over b_{k+2} while b_k, b_{k+1} and the
 * source are still in L2: five passes over a signal block per two steps instead of eight, and
 * the same bits as gsp_cheby_clenshaw_f32, since every row is computed by the same instructions.
 *
 * gsp_cheby_pair_plan_host: the slot tables, once per (matrix, rows_per_tile).  Pure host code
 *   on HOST copies of indptr / indices.  nbr_ptr (T + 1 entries, T = n / rows_per_tile) and
 *   nbr_idx list per tile the tiles its rows reference and the tile itself; slots_fwd / slots_rev
 *   (2 T entries each) are the launch orders of the two walk directions, (tile << 1) | step.  A
 *   second-step tile is placed `lag` first-step tiles after the last one it reads, so that it
 *   does not start while that one still runs on another CTA (the package passes 192: one
 *   wave of 396 CTAs is 396 slots, about 198 first-step tiles).
 *   *nbr_count_out receives the length of nbr_idx; when it exceeds nbr_capacity nothing else is
 *   written and the caller calls again with that much room.  Each table is checked to place
 *   every second-step tile after the first-step tiles it reads, else the call fails.
 * gsp_cheby_clenshaw_pairs_wanted: 1 when pairing pays for an (n, nsig) float32 block under this
 *   tile plan: the block exceeds the device's L2 (a block that fits is served from L2 by single
 *   steps already).  GSPB200_CLENSHAW_PAIRS=0 / 1 forces the answer (A/B measurements, tests).
 * gsp_cheby_clenshaw_pairs_f32: as gsp_cheby_clenshaw_f32 with nsrc = 1, but work holds
 *   3*n*nsig elements, plan_host must hold a tiling, the four tables are DEVICE copies of the
 *   plan, and tile_done is a device scratch array of T uint32 private to the call.  Every CTA of
 *   a paired launch must be resident at once (the grid is sized so); a second-step tile polls
 *   tile_done for a bounded time and traps if the first-step tiles it needs never finish. */
int gsp_cheby_pair_plan_host(int64_t n, const int32_t* indptr_host, const int32_t* indices_host,
                             int rows_per_tile, int lag, int64_t nbr_capacity, int32_t* nbr_ptr,
                             int32_t* nbr_idx, int32_t* slots_fwd, int32_t* slots_rev,
                             int64_t* nbr_count_out);
int gsp_cheby_clenshaw_pairs_wanted(int64_t n, int64_t nsig, const gsp_tile_plan* plan_host);

/* Neighbour rings of the tiled Clenshaw steps, once per (matrix, rows_per_tile).  The ring of tile
 * t (rows [t R, t R + R), t < T = n / R) is the sorted union of the tile's own rows and the
 * columns its rows reference.  A tiled step with a ring copies the tile's ring rows of the
 * gathered block into shared memory (one 1-D bulk copy per run of consecutive rows) and gathers
 * from there; the CSR slab then carries 16-bit ring positions instead of column ids.
 *
 * gsp_cheby_ring_plan_host: pure host code on HOST copies of indptr / indices.  Writes, per full
 *   tile, tile_meta[4 t .. 4 t + 4) = {first run, end of runs, ring rows, ring position of row
 *   t R}; per run, runs[2 i .. 2 i + 2) = {first row, ring position}; per stored entry j of a
 *   full tile, local[j] = the ring position of indices[j] (0 past the last full tile).
 *   *ring_max_out receives the rows of the largest ring, *run_count_out the number of runs; when
 *   that exceeds run_capacity, or the largest ring exceeds 65535 rows, only the two counts are
 *   written.
 * gsp_cheby_ring_fits: 1 when a ring of ring_max rows fits the shared memory of a tiled step of
 *   nsig signals under this tile plan, else 0 (GSPB200_TILE_RING=0 also gives 0: an A/B probe).
 * gsp_cheby_clenshaw_ring_f32: gsp_cheby_clenshaw_f32 (slots_fwd == NULL) or
 *   gsp_cheby_clenshaw_pairs_f32 (the pair tables given) with the rings of ring_host, whose
 *   pointers are device copies of the plan above for plan_host->rows_per_tile; ring_host may be
 *   NULL (no ring).  Same bits either way. */
typedef struct gsp_ring_plan {
  int rows_per_tile;
  int ring_max;
  const int32_t* tile_meta;
  const int32_t* runs;
  const uint16_t* local;
} gsp_ring_plan;
int gsp_cheby_ring_plan_host(int64_t n, const int32_t* indptr_host, const int32_t* indices_host,
                             int rows_per_tile, int64_t run_capacity, int32_t* tile_meta,
                             int32_t* runs, uint16_t* local, int64_t* run_count_out,
                             int32_t* ring_max_out);
int gsp_cheby_ring_fits(int ring_max, int64_t nsig, const gsp_tile_plan* plan_host);
int gsp_cheby_clenshaw_ring_f32(int64_t n, int64_t nnz, const int32_t* indptr,
                                const int32_t* indices, const float* data, double lmax,
                                const double* coeffs_host, int nsrc, int m, const float* sources,
                                int64_t nsig, float* out, float* work,
                                const gsp_tile_plan* plan_host, const gsp_ring_plan* ring_host,
                                const int32_t* slots_fwd, const int32_t* slots_rev,
                                const int32_t* nbr_ptr, const int32_t* nbr_idx,
                                uint32_t* tile_done, void* stream);
int gsp_cheby_clenshaw_pairs_f32(int64_t n, int64_t nnz, const int32_t* indptr,
                                 const int32_t* indices, const float* data, double lmax,
                                 const double* coeffs_host, int m, const float* source,
                                 int64_t nsig, float* out, float* work,
                                 const gsp_tile_plan* plan_host, const int32_t* slots_fwd,
                                 const int32_t* slots_rev, const int32_t* nbr_ptr,
                                 const int32_t* nbr_idx, uint32_t* tile_done, void* stream);

/* ------------------------------------------------------------------- lmax ---
 * gsp_spmv_*: y = L x for ONE vector -- scipy's csr_matvec, the product ARPACK calls at
 *   pygsp/graphs/graph.py:911-917 and the one of graph.py:955.  2..32 lanes per row (from the
 *   mean row length), coalesced reads of indices / data, warp-shuffle reduction per row.
 * gsp_lanczos_*: pygsp/graphs/graph.py:911-917 (scipy eigsh -> ARPACK).
 *   Runs Lanczos iterations [j0, j1) on L: two launches per iteration (the SpMV above with
 *   the v'Lv dot product fused in; the three-term update fused with the norm).  V3 holds
 *   3*n elements, scal_dev 2*cap+1+4096 doubles: alpha[0..cap) | beta[-1..cap) | reduction
 *   partials (beta[j] couples v_j and v_{j+1}; beta[-1] is the norm of the start vector).
 *   j0 == 0 seeds the start vector from `seed` (counter-based, reproducible).  The host
 *   reads alpha/beta back and diagonalises the tridiagonal matrix.
 */
int gsp_spmv_f32(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                 const float* data, const float* x, float* y, void* stream);
int gsp_spmv_f64(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                 const double* data, const double* x, double* y, void* stream);
int gsp_lanczos_f32(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                    const float* data, float* V3, int j0, int j1, int cap, uint64_t seed,
                    double* scal_dev, void* stream);
int gsp_lanczos_f64(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                    const double* data, double* V3, int j0, int j1, int cap, uint64_t seed,
                    double* scal_dev, void* stream);

/* ------------------------------------------------------------------ graph ---
 * gsp_coo_to_csr_*    graph.py:109  sparse.csr_matrix(coo): sort by (row, col), sum duplicates.
 *     indices / data are sized nnz by the caller; the number of distinct entries comes back
 *     in *n_unique_host_out (the call synchronises the stream once).
 * gsp_csr_inspect_*   graph.py:111-122  NaN / Inf / negative / self-loop checks.
 *     stats_dev[8] (int64): [0] NaN [1] Inf [2] negative [3] non-zero diagonal
 *     [4] stored zeros [5] unsorted-or-duplicate columns [6] column out of range.
 * gsp_csr_compact_*   graph.py:128      eliminate_zeros().
 * gsp_csr_asymmetry_* graph.py:403-405  (W != W.T).nnz: entries whose mirror differs.
 * gsp_csr_transpose_* W.T as sorted CSR (needed by the directed-graph branches).
 * gsp_csr_average_*   utils.py:247-248  (A + B)/2, exact zeros dropped.
 * gsp_degree_*        graph.py:772-781, 830-838  d and dw (pass the transpose for
 *     a directed graph, else NULL); d may be NULL.
 * gsp_laplacian_*     graph.py:618-628  lap_type 0 combinatorial, 1 normalized; the
 *     input must be the SYMMETRIC adjacency ((W+W.T)/2 for a directed graph).
 *     indptr/indices of the result are bit-identical to SciPy's.
 * gsp_spectral_bounds_* graph.py:939-958  out5_dev (double): max W, max dw,
 *     max(dw_s+dw_t) over edges, max(dw+(Ws dw)/dw), #NaN terms of the latter.
 * gsp_gather_rows_* / gsp_scatter_rows_*  dst[i,:] = src[idx[i],:] / dst[idx[i],:] = src[i,:]
 *     (vertex reordering in and out, halo packing).
 */
/* ----------------------------------------------------------------- solver ---
 * gsp_cg_*: conjugate gradients for (diag(row_scale) * tau * L + diag(diag)) X = B, a block
 *   of nsig <= 256 right-hand sides advancing together.  Stands for scipy.sparse.linalg.cg
 *   on the operator x -> M x + tau L x of pygsp/learning.py:326-337 (regression_tikhonov,
 *   one solve per column there) and, with row_scale = 1 - M, diag = 0, for the constrained
 *   problem of learning.py:350-365 restricted to the unlabelled vertices.  row_scale / diag
 *   are length-n vectors or NULL (= 1 / = 0).  Runs iterations [it0, it1) (it0 == 0 starts
 *   from X = 0); X, R, P, Q are (n, nsig) state blocks owned by the caller; scal_dev holds
 *   (cap + 1 + 2048) * nsig doubles, its first (cap + 1) x nsig entries are the history of
 *   the squared residual norms per column, which the host reads to test convergence. */
#define GSPB200_DECLARE_CG_API(SUF, T)                                                           \
  int gsp_cg_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,       \
                   const T* data, double tau, const T* row_scale, const T* diag, const T* B,     \
                   T* X, T* R, T* P, T* Q, int64_t nsig, int it0, int it1, int cap,              \
                   double* scal_dev, void* stream);

GSPB200_DECLARE_CG_API(f32, float)
GSPB200_DECLARE_CG_API(f64, double)

/* gsp_fb_simplex_*: accelerated forward-backward (FISTA) for
 *   min_X tau tr(X^T L X) + ||M (X - Y)||^2  s.t. every row of X on the probability simplex,
 *   Y the one-hot (n, nclass) matrix of the labels -- pyunlocbox's forward_backward + solve on the
 *   problem of pygsp/learning.py:42-180 (classification_tikhonov_simplex), started from X = Y.
 *   label (n, int32): class of a labelled vertex, -1 where M is False; 1 <= nclass <= 256.
 *   step: the gradient step (the reference's 0.5 / (1 + tau lmax)).  Runs iterations
 *   [it0, it1) (it0 == 0 writes X = Y and resets the state); an iteration is the SpMM L X_k
 *   (gsp_cheby_step_*, tiled where plan_host applies) and one row pass that forms the
 *   extrapolated point, its gradient (L y by linearity: no second SpMM), projects every row onto
 *   the simplex (Michelot, sort-free) and adds up the objective of X_k in a fixed order.  X2 and
 *   LX2 each hold two (n, nclass) row-major blocks; iterate k is X2 block k % 2.
 *   Stop tests of pyunlocbox.solvers.solve, on iterate k >= 1 with objective f_k:
 *   tol_host = {atol, dtol, rtol, xtol} (host doubles, NaN = off), maxit < 0 = off;
 *   f_k < atol | |f_k - f_{k-1}| < dtol | |f_k - f_{k-1}| / |f_k| < rtol (f_{k-1} when f_k = 0,
 *   ratio 0 when both are) | ||X_k - X_{k-1}|| / sqrt(n nclass) < xtol | k >= maxit; the last
 *   one that holds names the stop.  Once one holds, later row passes do nothing, so the state
 *   stays at the stopping iterate however far past it the caller enqueued.  scal_dev holds
 *   GSPB200_FB_HISTORY + cap doubles (it1 <= cap): [1] the stop criterion (0 = running,
 *   1 atol, 2 dtol, 3 rtol, 4 xtol, 5 maxit), [2] the stop iteration, and from
 *   GSPB200_FB_HISTORY on the objective f_k of every iterate, which the host reads. */
#define GSPB200_FB_HISTORY 3080
#define GSPB200_DECLARE_FB_API(SUF, T)                                                           \
  int gsp_fb_simplex_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices, \
                           const T* data, const int32_t* label, int64_t nclass, double tau,       \
                           double step, const double* tol_host, int maxit, T* X2, T* LX2,         \
                           int it0, int it1, int cap, double* scal_dev,                           \
                           const gsp_tile_plan* plan_host, void* stream);

GSPB200_DECLARE_FB_API(f32, float)
GSPB200_DECLARE_FB_API(f64, double)

/* Graph total variation prox, min_z 1/2 ||x - z||^2 + gamma ||D^T A z||_1, by FISTA on the dual
 * (csrc/tv.cu): pygsp/optimization.py:24-103 (prox_tv), which hands the problem to pyunlocbox's
 * norm_l1 prox (:100-103) and cannot run as written.  D is the (n x n_edges) differential operator
 * and Dt its transpose (csrc/difference.cu: two entries per Dt row, none for a self-loop).
 * Blocks are row-major with nsig columns.  The caller owns the state and zero-fills it before
 * iteration 0: U2 holds two dual blocks of max(n, n_edges) rows (u_k is block k % 2; the rows
 * past n_edges stay zero), G one (n_edges, nsig) block (g_k = D^T A z_k), scal_dev
 * GSPB200_TV_HISTORY + 2 cap doubles: [0] t_k, [1] the stop criterion (0 = running, 1 rtol,
 * 2 maxit), [2] the stop iteration, then P_k = 1/2 ||x - z_k||^2 + gamma ||g_k||_1 at
 * GSPB200_TV_HISTORY + 2 k and gap_k = gamma sum(|g_k| - u_k g_k) at GSPB200_TV_HISTORY + 2 k + 1
 * (appending zeros between calls grows cap).
 * Stop rule on k >= 1 (optimization.py:53-57): |P_k - P_{k-1}| < tol |P_k|, or
 * P_k = P_{k-1} = 0 with tol > 0 (rtol); k >= maxit (maxit, checked second).  Once it holds the
 * edge passes do nothing, so u_k of the stopping iteration stays in U2; z does not (see
 * gsp_prox_tv_primal_*).  tau is the dual step 1 / (gamma nu_bar), nu_bar >= ||D^T A||^2.
 * gsp_prox_tv_*: iterations [it0, it1) of the A = identity path (it1 <= cap), each a vertex pass
 *     z = x - gamma D u_k (replaces l1_at, :89-90 / :97-98) and an edge pass.
 * gsp_prox_tv_edges_*: the edge pass of iteration it alone, for an A given by the caller: forms
 *     g_k = D^T w from w = A z_k (replaces l1_a, :86-87 / :94-95), z = z_k enters the objective.
 * gsp_prox_tv_primal_*: z = x - gamma D u for one dual block u of max(n, n_edges) rows: the
 *     vertex pass of gsp_prox_tv_*, bit for bit (z_k of the stopping iteration from u_k). */
#define GSPB200_TV_HISTORY 3080
#define GSPB200_DECLARE_TV_API(SUF, T)                                                           \
  int gsp_prox_tv_##SUF(int64_t n, int64_t n_edges, int64_t d_nnz, const int32_t* d_indptr,     \
                        const int32_t* d_indices, const T* d_data, const int32_t* dt_indptr,    \
                        const int32_t* dt_indices, const T* dt_data, const T* x, int64_t nsig,  \
                        double gamma, double tau, double tol, int maxit, T* z, T* U2, T* G,     \
                        int it0, int it1, int cap, double* scal_dev, void* stream);             \
  int gsp_prox_tv_edges_##SUF(int64_t n, int64_t n_edges, const int32_t* dt_indptr,             \
                              const int32_t* dt_indices, const T* dt_data, const T* w,          \
                              const T* x, const T* z, int64_t nsig, double gamma, double tau,   \
                              double tol, int maxit, T* U2, T* G, int it, int cap,              \
                              double* scal_dev, void* stream);                                  \
  int gsp_prox_tv_primal_##SUF(int64_t n, int64_t d_nnz, const int32_t* d_indptr,               \
                               const int32_t* d_indices, const T* d_data, const T* x,           \
                               int64_t nsig, double gamma, const T* u, T* z, void* stream);

GSPB200_DECLARE_TV_API(f32, float)
GSPB200_DECLARE_TV_API(f64, double)

/* --------------------------------------------------------- spectral basis ---
 * Tall-skinny block kernels of the graph Fourier basis (pygsp_b200/graphs/fourier.py): gft /
 * igft and the partial eigensolver that stands for scipy's eigsh (Chebyshev-filtered subspace
 * iteration; its filter is gsp_cheby_step_* with nscales = 0).  Blocks are row-major (n, k)
 * float / double; the small matrices C, Q and the vectors theta, out are double, row-major.
 * Sums over rows accumulate in double and run in a fixed order that depends on the shapes
 * only, so the results are bit-reproducible.  Scratch is stream-ordered (cudaMallocAsync).
 * gsp_block_gram_*: C (ka x kb) = A^T B for A (n x ka), B (n x kb); C must not overlap A or B.
 *   np.tensordot(U, s, ([0], [0])) of gft (pygsp/graphs/fourier.py:229-230), and the Gram
 *   and projected matrices that ARPACK forms inside eigsh (fourier.py:175).
 * gsp_block_combine_*: Y (n x kq) = A Q for A (n x ka), Q (ka x kq); Y must not overlap A.
 *   np.tensordot(U, s_hat, ([1], [0])) of igft (fourier.py:264), and the basis updates of eigsh.
 * gsp_block_residual_*: out[j] = ||LX[:, j] - theta[j] X[:, j]||^2 for X, LX (n x k) -- the
 *   residual norms eigsh tests for convergence (fourier.py:175).
 * gsp_block_random_*: X[i] = uniform [-1, 1) of (seed, i) for the n*k entries of X -- the
 *   eigensolver's start block, counter-based like gsp_lanczos_*'s start vector.
 */
#define GSPB200_DECLARE_BLOCK_API(SUF, T)                                                        \
  int gsp_block_gram_##SUF(int64_t n, const T* A, int64_t ka, const T* B, int64_t kb, double* C, \
                           void* stream);                                                        \
  int gsp_block_combine_##SUF(int64_t n, const T* A, int64_t ka, const double* Q, int64_t kq,    \
                              T* Y, void* stream);                                               \
  int gsp_block_residual_##SUF(int64_t n, const T* X, const T* LX, const double* theta,          \
                               int64_t k, double* out, void* stream);                            \
  int gsp_block_random_##SUF(int64_t n, int64_t k, uint64_t seed, T* X, void* stream);

GSPB200_DECLARE_BLOCK_API(f32, float)
GSPB200_DECLARE_BLOCK_API(f64, double)

/* ------------------------------------------------------- Lanczos filtering ---
 * Per-signal Krylov bases of pygsp/filters/approximations.py:228-341 (lanczos_op, lanczos):
 * one independent Lanczos process per column of a row-major (n, nsig) block, with full
 * reorthogonalisation against that column's own basis.  Columns never mix, and every sum over
 * rows accumulates in double over a row partition that depends on n only, so a column's bits do
 * not depend on nsig or on the other columns.  Scratch is stream-ordered (cudaMallocAsync).
 * gsp_krylov_basis_*: A is n x ncols CSR and must be square (ncols != n is refused before any
 *   launch: the SpMM reads the basis at A's column indices).  V is (order + 1, n, nsig)
 *   (vector k of column j is V[k, :, j]; slot order is workspace).  On return, for every column j (arrays of double, row-major, on the device):
 *   alpha (order x nsig) the diagonal of T_j, beta (order x nsig) its off-diagonal
 *   (beta[k] = beta_k couples vectors k - 1 and k; beta[0] = ||x_j||), vs (order x nsig) = V^T x
 *   and m (nsig, int32) the Krylov dimension.  A column stops growing (breakdown) when
 *   beta_{k+1} <= 16 eps max(largest |alpha|, |beta| so far, ||A||_inf); its vectors past m and
 *   its alpha, beta past the leading m x m block are zero.  A zero column has m = 0.
 * gsp_krylov_combine_*: Y[f, r, j] = sum_{i < k} V[i, r, j] W[f, i, j] for W (nf, k, nsig)
 *   double; Y is (nf, n, ldy) with ldy >= nsig (a column range of a wider block).  One pass
 *   over V for up to 16 filters.
 */
#define GSPB200_DECLARE_KRYLOV_API(SUF, T)                                                       \
  int gsp_krylov_basis_##SUF(int64_t n, int64_t ncols, const int32_t* indptr,                   \
                             const int32_t* indices,                                             \
                             const T* data, const T* x, int64_t nsig, int order, T* V,           \
                             double* alpha, double* beta, double* vs, int32_t* m, void* stream); \
  int gsp_krylov_combine_##SUF(int64_t n, const T* V, int64_t k, const double* W, int64_t nf,   \
                               int64_t nsig, T* Y, int64_t ldy, void* stream);

GSPB200_DECLARE_KRYLOV_API(f32, float)
GSPB200_DECLARE_KRYLOV_API(f64, double)

/* ---------------------------------------------------------------- features ---
 * pygsp/features.py without the frame (pygsp_b200/features.py).  The squared row norms of the
 * frame, ||p(L) e_i||^2 for p = c0/2 T_0 + sum_k c_k T_k(Lt), Lt = 2 L / lmax - I, are
 * sum_n d_n mu_n(i) with mu_n(i) = (T_n(Lt))_ii and d the Chebyshev series of p^2; one
 * recurrence over identity probe blocks gives mu for every kernel.  The blocks T_k are produced
 * by gsp_cheby_step_* (nscales = 0; first step alpha = 2/lmax, beta = -1; then alpha = 4/lmax,
 * beta = -2, gamma = -1).
 * gsp_probe_block_*: X (n, b) row-major = columns v0 .. v0 + b - 1 of the identity -- the
 *   s = np.identity(N) that compute_frame filters (pygsp/filters/filter.py:599), b columns at a
 *   time.
 * gsp_cheby_moments_step_*: after step k (t_next = T_{k+1}, t_cur = T_k, both (n, b)), writes
 *   sums[k][0][j] = sum_r t_next[r, j]^2 and sums[k][1][j] = sum_r t_next[r, j] t_cur[r, j] into
 *   sums (m, 2, b) double.  Sums accumulate in double over a row partition that depends on n
 *   only, so column j's sums do not depend on b or on the other columns.
 * gsp_cheby_moments_finish: mu rows v0 .. v0 + b - 1 of mu (n, 2m + 1) double from sums after
 *   the m steps: mu_0 = 1, mu_1 = sums[0][1], mu_{2k} = 2 sums[k-1][0] - 1,
 *   mu_{2k+1} = 2 sums[k][1] - mu_1.  Stands for np.linalg.norm(tig, axis=1) of
 *   compute_norm_tig (pygsp/features.py:58-59), with the atom combination done by
 *   gsp_block_combine_f64.
 * gsp_two_hop_count_*: np.dot(G.A, G.A) with G.A = W > 0 (pygsp/features.py:23,
 *   graph.py:718-727), a boolean product: two_hop[i] = number of distinct c with W[i, k] > 0 and
 *   W[k, c] > 0 for some k; degree[i] = number of k with W[i, k] > 0 (np.sum(G.A, axis=1)).
 *   Exact for any degree distribution; scratch is bounded (heavy rows are processed in chunks).
 *   The call synchronises `stream` (once, and once per chunk of heavy rows).
 */
#define GSPB200_DECLARE_MOMENTS_API(SUF, T)                                                      \
  int gsp_probe_block_##SUF(int64_t n, int64_t v0, int64_t b, T* X, void* stream);              \
  int gsp_cheby_moments_step_##SUF(int64_t n, const T* t_next, const T* t_cur, int64_t b, int m, \
                                   int k, double* sums, void* stream);                           \
  int gsp_two_hop_count_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,         \
                              const T* data, int32_t* two_hop, int32_t* degree, void* stream);

GSPB200_DECLARE_MOMENTS_API(f32, float)
GSPB200_DECLARE_MOMENTS_API(f64, double)

int gsp_cheby_moments_finish(int64_t n, int m, int64_t v0, int64_t b, const double* sums,
                             double* mu, void* stream);

/* ------------------------------------------------- host <-> device staging ---
 * Filter.filter() takes and returns host arrays (filter.py:146-328).  To overlap the PCIe
 * transfers with the recurrence the signal block is processed in COLUMN chunks; a chunk of a
 * row-major (n, nsig) block is a strided 2-D region (`height` rows of `width_bytes`, row
 * pitches in bytes).
 * gsp_copy2d_async: cudaMemcpy2DAsync on `stream` (copy engines); kind 1 = host to device,
 *   2 = device to host, 3 = device to device.  Host memory must be page-locked.
 * gsp_stage_cols: the same region moved by a kernel of at most max_blocks blocks (0 = one
 *   per SM) that reads / writes PINNED host memory through its unified address; all
 *   pointers, pitches and width_bytes must be multiples of 16. */
int gsp_copy2d_async(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width_bytes,
                     size_t height, int kind, void* stream);
int gsp_stage_cols(void* dst, size_t dpitch, const void* src, size_t spitch, size_t width_bytes,
                   size_t height, int max_blocks, void* stream);

/* ------------------------------------------------------------ peer-memory halo ---
 * The vertex-partitioned path (no reference counterpart: PyGSP is single-process).
 * gsp_ipc_alloc / open / close / free: cudaMalloc'ed, zero-filled buffers exported with
 *     CUDA IPC (64-byte handle) so that the other ranks of the node can map them.
 * gsp_halo_push_*: copies rows src[src_row[e], :] into peer_base[dst_peer[e]][dst_row[e], :]
 *     (peer stores over NVLink), fences, then writes `value` to every peer_flags[q]
 *     (the address of this rank's slot in neighbour q's flag array).
 *     done_counter: one zero-initialised device uint32 owned by the caller.
 * gsp_halo_wait: blocks the STREAM (not the host) until flags[neighbor_ids[q]] >= value.
 */
int gsp_ipc_alloc(size_t bytes, void** dev_ptr_out, unsigned char* handle64_out);
int gsp_ipc_open(const unsigned char* handle64, void** dev_ptr_out);
int gsp_ipc_close(void* dev_ptr);
int gsp_ipc_free(void* dev_ptr);
int gsp_halo_push_f32(int64_t n_send, const int64_t* src_row, const int32_t* dst_peer,
                      const int64_t* dst_row, const float* src, float* const* peer_base,
                      int64_t width, uint64_t* const* peer_flags, int n_neighbors,
                      uint64_t value, uint32_t* done_counter, void* stream);
int gsp_halo_push_f64(int64_t n_send, const int64_t* src_row, const int32_t* dst_peer,
                      const int64_t* dst_row, const double* src, double* const* peer_base,
                      int64_t width, uint64_t* const* peer_flags, int n_neighbors,
                      uint64_t value, uint32_t* done_counter, void* stream);
int gsp_halo_wait(const uint64_t* flags, const int32_t* neighbor_ids, int n_neighbors,
                  uint64_t value, void* stream);

/* ------------------------------------------- the partitioned operator, one call ---
 * gsp_cheby_op_dist_*: approximations.py:58-114 on ONE rank's row block of a 1-D vertex
 * partitioned Laplacian (SURVEY.md 8e).  The caller (one process per GPU) builds the plan
 * once -- which of its rows every neighbour needs and where they live in the neighbour's
 * halo, the CUDA-IPC mapped state buffers and flag arrays; that is host-side set-up and
 * needs the job's communicator once (pygsp_b200/distributed.py: HaloPlan, PeerWindow) --
 * and then runs any number of calls without any collective: each of the K recurrence
 * steps waits for the neighbours' flags, computes, stores its boundary rows into the
 * neighbours' halo rows over NVLink and publishes the step (all inside the fused step
 * kernel for float32 with a tile plan; wait / step / push kernels otherwise).
 *
 *   local rows are ordered boundary-first (rows [0, n_boundary_rows) reference halo
 *   columns, rows [0, n_push_rows) are needed by neighbours); local column j < n_local is
 *   local row j, column n_local + h is halo slot h.
 *   buf[b]        : this rank's state buffers, (n_local + n_halo, nsig) each, inside its IPC
 *                   window; buf[2] may be NULL (then the Clenshaw form is not used)
 *   peer_base[b]  : device array of P pointers, entry q = rank q's buf[b] (mapped)
 *   peer_flags[i] : device array, entry i = address of THIS rank's slot in the flag array
 *                   of neighbour neighbor_ids[i]; flags = this rank's own flag array (P slots)
 *   src_row/dst_peer/dst_row (n_send entries): the rows to push as a flat list;
 *   push_ptr/push_peer/push_row: the same list as a CSR over local rows [0, n_push_rows)
 *   push_counter / fused_counter: zero-initialised device counters owned by the caller
 *   x : (n_local, nsig) input (NULL: already in buf[0], local order);
 *   r : (nscales, n_local, nsig) output; x and r are in the CALLER's row order when
 *       plan->perm is given (the gather into local order replaces the copy into buf[0]; the
 *       Clenshaw form stores its last step straight to the caller's rows), else local order;
 *   clenshaw != 0 and nscales == 1: backward (Clenshaw) recurrence, one pass less per order;
 *   seq_host : the rank's sequence counter (starts at 0, advanced by m + 2 per call; all
 *              ranks must make the same calls in the same order).
 * Everything is enqueued on `stream`; nothing synchronises. */
typedef struct gsp_dist_plan {
  int64_t n_local, n_halo, nnz;
  const int32_t* indptr;
  const int32_t* indices;
  const void* data;                  /* float / double values of the local CSR */
  void* buf[3];
  void* const* peer_base[3];
  uint64_t* const* peer_flags;
  uint64_t* flags;
  const int32_t* neighbor_ids;
  int32_t n_neighbors;
  int32_t separate_exchange; /* != 0: never fuse the exchange into the step kernel (wait / step / push kernels) */
  uint32_t* push_counter;
  uint64_t* fused_counter;
  int64_t n_send;
  const int64_t* src_row;
  const int32_t* dst_peer;
  const int64_t* dst_row;
  int64_t n_push_rows;
  const int32_t* push_ptr;
  const int32_t* push_peer;
  const int64_t* push_row;
  int64_t n_boundary_rows;
  const int64_t* perm;               /* local row i = row perm[i] of the caller's blocks; NULL: identity */
} gsp_dist_plan;

int gsp_cheby_op_dist_f32(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                          double lmax, const double* coeffs_host, int nscales, int m, const float* x,
                          int64_t nsig, float* r, int clenshaw, uint64_t* seq_host, void* stream);
int gsp_cheby_op_dist_f64(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                          double lmax, const double* coeffs_host, int nscales, int m, const double* x,
                          int64_t nsig, double* r, int clenshaw, uint64_t* seq_host, void* stream);

/* gsp_cheby_op_dist_phases_*: the same call cut into its m + 1 phases; enqueues phases
 * [phase_begin, phase_end) only (gsp_cheby_op_dist_* is the range [0, m + 1)).  Each phase
 * first waits, then pushes, so that several ranks can share one device and one stream when the
 * caller runs phase j of every rank before phase j + 1 of any (base = *seq_host as passed in):
 *   phase 0      entry barrier: publishes base+1, waits for nothing
 *   phase 1      waits for base+1, brings in x (gather by perm, or copy), publishes base+2
 *   phase 1 + s  recurrence step s = 1 .. m-1 (forward or Clenshaw): waits for base+1+s and
 *                publishes base+2+s, except the last step, which publishes nothing
 * The blocks a phase reads and writes depend on the phase alone.  *seq_host advances by m + 2
 * only when phase_end == m + 1.  A forward-form range that is not the whole call refuses
 * plan->perm (its accumulators are call-local then) with an error, before any launch. */
int gsp_cheby_op_dist_phases_f32(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                                 double lmax, const double* coeffs_host, int nscales, int m,
                                 const float* x, int64_t nsig, float* r, int clenshaw,
                                 uint64_t* seq_host, int phase_begin, int phase_end, void* stream);
int gsp_cheby_op_dist_phases_f64(const gsp_dist_plan* plan_host, const gsp_tile_plan* tile_host,
                                 double lmax, const double* coeffs_host, int nscales, int m,
                                 const double* x, int64_t nsig, double* r, int clenshaw,
                                 uint64_t* seq_host, int phase_begin, int phase_end, void* stream);

/* ------------------------------------------------------ on-device graph construction ---
 * gsp_grid2d_*: adjacency of pygsp/graphs/grid2d.py:40-89 (n1 x n2 grid, 4 neighbours, unit
 *     weights, row-major numbering) as canonical CSR; count writes indptr (n1*n2 + 1).
 * gsp_knn_grid: k nearest neighbours (self excluded) of n points in 2-D / 3-D by a
 *     uniform cell grid -- the scipy.spatial.KDTree query of nngraph.py:213-216 for the
 *     Euclidean metric; other dimensions and metrics: gsp_knn_brute below.
 *     points (n, dim) double; lo/hi: bounding box (finite), cells: grid resolution, 1 .. 2^30
 *     per axis and < 2^31 in all (host arrays of length dim); outputs (n, k) row-major,
 *     ascending distance, ties by index: the lists of gsp_knn_brute(p = 2), bit for bit.
 * gsp_knn_to_csr_*: directed k-NN matrix W[i, nn] = exp(-d^2/sigma) as CSR with sorted
 *     rows (nngraph.py:221-226,289); symmetrise with gsp_csr_transpose / _average.
 */
int gsp_grid2d_count(int64_t n1, int64_t n2, int32_t* indptr, int64_t* nnz, void* stream);
int gsp_grid2d_fill_f32(int64_t n1, int64_t n2, const int32_t* indptr, int32_t* indices,
                        float* data, void* stream);
int gsp_grid2d_fill_f64(int64_t n1, int64_t n2, const int32_t* indptr, int32_t* indices,
                        double* data, void* stream);
int gsp_knn_grid(int64_t n, int dim, const double* points, int k, const double* lo_host,
                 const double* hi_host, const int32_t* cells_host, int32_t* nn_idx,
                 double* nn_dist, void* stream);
int gsp_knn_to_csr_f32(int64_t n, int k, const int32_t* nn_idx, const double* nn_dist,
                       double sigma, int32_t* indptr, int32_t* indices, float* data, void* stream);
int gsp_knn_to_csr_f64(int64_t n, int k, const int32_t* nn_idx, const double* nn_dist,
                       double sigma, int32_t* indptr, int32_t* indices, double* data,
                       void* stream);

/* ----------------------------------------------------- neighbour search, any dimension ---
 * Exhaustive search over n points of dimension d >= 1 (points (n, d) row-major double), in the
 * Minkowski metric of order p: p = 1 (manhattan), 2 (euclidean), INFINITY (max_dist) or any
 * p >= 1 (minkowski: (sum |x_i - y_i|^p)^(1/p)); nngraph.py:162-167's dist_translation.  The
 * difference is accumulated in dimension order, in double, and the root is taken once (as
 * cKDTree).  Self is excluded by index, never by position.  csrc/neighbors.cu.
 * gsp_knn_brute: nngraph.py:213-216, KDTree(X).query(X, k + 1, p) without the self column, for
 *     any d.  1 <= k <= 32, k < n.  Outputs (n, k) like gsp_knn_grid: ascending (distance, id),
 *     independent of the launch configuration.
 * gsp_radius_count / gsp_radius_fill_f64: nngraph.py:228-283, query_ball_point(r = epsilon, p)
 *     and the j != i filter: row i = {j != i : dist(x_i, x_j) <= epsilon}.  fill writes the
 *     columns (sorted, bit-identical from run to run) and their distances (double).
 * gsp_csr_symmetrize_count_* / _fill_*: utils.py:244-277 symmetrize(W, method) for mode
 *     0 'maximum' (W - W o [W^T > W] + W^T o [W^T > W]), 1 'fill' (W + ((A + A^T) - A) o W^T,
 *     A = W > 0, then 'average'), 2 'tril' and 3 'triu' (one triangle, then 'maximum').  A is W,
 *     B = W^T (gsp_csr_transpose_*); exact zeros are dropped.  'average' is gsp_csr_average_*.
 * gsp_gauss_weights_*: w = exp(-d^2 / sigma) for nnz distances (nngraph.py:276-281).
 */
int gsp_knn_brute(int64_t n, int d, const double* points, int k, double p, int32_t* nn_idx,
                  double* nn_dist, void* stream);
int gsp_radius_count(int64_t n, int d, const double* points, double epsilon, double p,
                     int32_t* indptr, int64_t* nnz, void* stream);
int gsp_radius_fill_f64(int64_t n, int d, const double* points, double epsilon, double p,
                        const int32_t* indptr, int32_t* indices, double* dist, void* stream);
/* Segmented search: the vertices form n_seg contiguous segments, seg_start (n_seg + 1 int64,
 * device) non-decreasing from 0 to n, and seg_id (n int32, device) the segment of every vertex
 * (seg_start[seg_id[i]] <= i < seg_start[seg_id[i] + 1]).  Query i sees only the candidates of
 * its own segment: the result is the unsegmented search of each segment alone, ids offset by
 * the segment start, bit for bit.  The work is about the sum of the squared segment sizes.
 * gsp_knn_brute_seg: 1 <= k <= 32; a vertex whose segment has fewer than k other points gets
 *     its list padded with id -1 and distance 0. */
int gsp_knn_brute_seg(int64_t n, int d, const double* points, int k, double p, int64_t n_seg,
                      const int64_t* seg_start, const int32_t* seg_id, int32_t* nn_idx,
                      double* nn_dist, void* stream);
int gsp_radius_count_seg(int64_t n, int d, const double* points, double epsilon, double p,
                         int64_t n_seg, const int64_t* seg_start, const int32_t* seg_id,
                         int32_t* indptr, int64_t* nnz, void* stream);
int gsp_radius_fill_seg_f64(int64_t n, int d, const double* points, double epsilon, double p,
                            int64_t n_seg, const int64_t* seg_start, const int32_t* seg_id,
                            const int32_t* indptr, int32_t* indices, double* dist,
                            void* stream);

#define GSPB200_DECLARE_NEIGHBOR_API(SUF, T)                                                     \
  int gsp_csr_symmetrize_count_##SUF(int64_t n, int mode, const int32_t* a_indptr,               \
                                     const int32_t* a_indices, const T* a_data,                  \
                                     const int32_t* b_indptr, const int32_t* b_indices,          \
                                     const T* b_data, int32_t* s_indptr, int64_t* nnz,           \
                                     void* stream);                                              \
  int gsp_csr_symmetrize_fill_##SUF(int64_t n, int mode, const int32_t* a_indptr,                \
                                    const int32_t* a_indices, const T* a_data,                   \
                                    const int32_t* b_indptr, const int32_t* b_indices,           \
                                    const T* b_data, const int32_t* s_indptr,                    \
                                    int32_t* s_indices, T* s_data, void* stream);                \
  int gsp_gauss_weights_##SUF(int64_t nnz, const double* dist, double sigma, T* w, void* stream);

GSPB200_DECLARE_NEIGHBOR_API(f32, float)
GSPB200_DECLARE_NEIGHBOR_API(f64, double)

/* ---------------------------------------------------------------- spring layout ---
 * Fruchterman-Reingold force-directed layout of pygsp/graphs/_layout.py:169-219 on the device,
 * in float64 whatever the type of W (csrc/layout.cu).  pos / pos_in / pos_out / states are
 * (n, dim) row-major double blocks; W is canonical CSR (n x n) and only its entries with w > 0
 * attract (the reference's A = W > 0, graph.py:718, row i of a directed W); fixed (n bytes, may
 * be NULL) marks vertices that do not move but still repel (_layout.py:198).  One iteration:
 *   disp_i = sum_j delta_ij k^2 / d_ij^2 - sum_{j : w_ij > 0} delta_ij d_ij / k,
 *   delta_ij = p_i - p_j, d_ij = max(|delta_ij|, 0.01),           (_layout.py:200-211)
 *   p_i += disp_i t / length_i, length_i = |disp_i|, 0.1 if < 0.01  (_layout.py:212-215).
 * The sums run in a fixed order that depends on n only: results are bit-identical from run to
 * run and from card to card, and differ from the reference's order by rounding.
 * gsp_spring_step_*:   one iteration at temperature t from pos_in into pos_out (distinct
 *     blocks).
 * gsp_spring_layout_*: `iterations` iterations (_layout.py:194-217) from the start in pos, at
 *     temperatures temps_host[0 .. iterations) (host array; the caller's cooling schedule,
 *     _layout.py:190-191, 217); the final positions are written back to pos.  states (may be
 *     NULL; iterations x n x dim) receives the positions after every iteration.
 */
#define GSPB200_DECLARE_LAYOUT_API(SUF, T)                                                       \
  int gsp_spring_step_##SUF(int64_t n, int dim, const int32_t* indptr, const int32_t* indices,   \
                            const T* data, double k, double t, const uint8_t* fixed,             \
                            const double* pos_in, double* pos_out, void* stream);                \
  int gsp_spring_layout_##SUF(int64_t n, int dim, const int32_t* indptr, const int32_t* indices, \
                              const T* data, double k, int iterations, const double* temps_host, \
                              const uint8_t* fixed, double* pos, double* states, void* stream);

GSPB200_DECLARE_LAYOUT_API(f32, float)
GSPB200_DECLARE_LAYOUT_API(f64, double)

#define GSPB200_DECLARE_GRAPH_API(SUF, T)                                                        \
  int gsp_csr_inspect_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,            \
                            const T* data, int64_t* stats_dev, void* stream);                    \
  int gsp_csr_compact_count_##SUF(int64_t n, const int32_t* indptr, const T* data,               \
                                  int32_t* out_indptr, int64_t* nnz, void* stream);              \
  int gsp_csr_compact_fill_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,       \
                                 const T* data, const int32_t* out_indptr, int32_t* out_indices, \
                                 T* out_data, void* stream);                                     \
  int gsp_csr_asymmetry_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,          \
                              const T* data, int64_t* count_dev, void* stream);                  \
  int gsp_csr_transpose_##SUF(int64_t n, int64_t nnz, const int32_t* indptr,                     \
                              const int32_t* indices, const T* data, int32_t* t_indptr,          \
                              int32_t* t_indices, T* t_data, void* stream);                      \
  int gsp_coo_to_csr_##SUF(int64_t n, int64_t nnz, const int32_t* rows, const int32_t* cols,      \
                           const T* vals, int32_t* indptr, int32_t* indices, T* data,             \
                           int64_t* n_unique_host_out, void* stream);                            \
  int gsp_csr_average_count_##SUF(int64_t n, const int32_t* a_indptr, const int32_t* a_indices,  \
                                  const T* a_data, const int32_t* b_indptr,                      \
                                  const int32_t* b_indices, const T* b_data, int32_t* s_indptr,  \
                                  int64_t* nnz, void* stream);                                   \
  int gsp_csr_average_fill_##SUF(int64_t n, const int32_t* a_indptr, const int32_t* a_indices,   \
                                 const T* a_data, const int32_t* b_indptr,                       \
                                 const int32_t* b_indices, const T* b_data,                      \
                                 const int32_t* s_indptr, int32_t* s_indices, T* s_data,         \
                                 void* stream);                                                  \
  int gsp_degree_##SUF(int64_t n, const int32_t* indptr, const T* data,                          \
                       const int32_t* t_indptr, const T* t_data, double* dw, double* d,          \
                       void* stream);                                                            \
  int gsp_laplacian_count_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,        \
                                const T* data, const double* dw, int lap_type,                   \
                                int32_t* l_indptr, int64_t* nnz, void* stream);                  \
  int gsp_laplacian_fill_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,         \
                               const T* data, const double* dw, int lap_type,                    \
                               const int32_t* l_indptr, int32_t* l_indices, T* l_data,           \
                               void* stream);                                                    \
  int gsp_spectral_bounds_##SUF(int64_t n, const int32_t* w_indptr, const int32_t* w_indices,    \
                                const T* w_data, const int32_t* s_indptr,                        \
                                const int32_t* s_indices, const T* s_data, const double* dw,     \
                                double* out5_dev, void* stream);                                 \
  int gsp_gather_rows_##SUF(int64_t rows, const int64_t* idx, const T* src, int64_t width,       \
                            T* dst, void* stream);                                               \
  int gsp_scatter_rows_##SUF(int64_t rows, const int64_t* idx, const T* src, int64_t width,      \
                             T* dst, void* stream);

GSPB200_DECLARE_GRAPH_API(f32, float)
GSPB200_DECLARE_GRAPH_API(f64, double)

/* -------------------------------------------------------- differential operator ---
 * pygsp/graphs/difference.py:144-166 and graph.py:1019-1029, built on the device from a
 * canonical CSR adjacency W (n x n).  Edges are numbered in row-major CSR order: the entries
 * with col >= row (self-loops included) of an undirected W, every entry of a directed one.
 * D is the n x Ne incidence matrix (CSR), Dt = D^T (Ne x n, CSR; its arrays are the CSC arrays
 * of the reference's D).  A self-loop is an edge with an empty row of Dt (the reference's two
 * entries cancel and eliminate_zeros() drops them), so nnz(D) = 2 (Ne - loops); the caller
 * checks nnz(D) < 2^31 before allocating.  Values in double, rounded once: combinatorial
 * -+sqrt(w), normalized -sqrt(w / dw[s]) / +sqrt(w / dw[t]), divided by sqrt(2) if directed.
 * gsp_edge_offsets:     eptr (n + 1) = scan of each row's entries with col >= row (undirected;
 *     a directed graph's edge offsets are W's indptr).
 * gsp_edge_list_*:      sparse.triu(W, format='coo') / W.tocoo() (graph.py:1019-1026): sources,
 *     targets (int32) and weights (n_edges each), and Dt's indptr (n_edges + 1).
 * gsp_incidence_t_fill_*: Dt's indices / data (difference.py:147-166); dw (double) is the
 *     weighted degree the Laplacian uses; directed != 0 adds the 1/sqrt(2).
 * gsp_incidence_count / gsp_incidence_fill_*: D = Dt.T as CSR (the reference's D.tocsr()), each
 *     row in increasing edge id, without a sort; t_indptr / t_indices / t_data is W^T as sorted
 *     CSR for a directed graph, NULL for an undirected one; eptr as above (W's indptr if
 *     directed).
 * grad and div are gsp_spmm_* on Dt and D (difference.py:244, 331).
 */
int gsp_edge_offsets(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* eptr,
                     void* stream);
int gsp_incidence_count(int64_t n, const int32_t* indptr, const int32_t* indices,
                        const int32_t* t_indptr, const int32_t* t_indices, int32_t* d_indptr,
                        int64_t* nnz, void* stream);

#define GSPB200_DECLARE_DIFF_API(SUF, T)                                                         \
  int gsp_edge_list_##SUF(int64_t n, int64_t n_edges, const int32_t* indptr,                     \
                          const int32_t* indices, const T* data, const int32_t* eptr,            \
                          int32_t* sources, int32_t* targets, T* weights, int32_t* dt_indptr,    \
                          void* stream);                                                         \
  int gsp_incidence_t_fill_##SUF(int64_t n_edges, const int32_t* sources,                        \
                                 const int32_t* targets, const T* weights, const double* dw,     \
                                 int lap_type, int directed, const int32_t* dt_indptr,           \
                                 int32_t* dt_indices, T* dt_data, void* stream);                 \
  int gsp_incidence_fill_##SUF(int64_t n, int lap_type, const int32_t* indptr,                   \
                               const int32_t* indices, const T* data, const int32_t* eptr,       \
                               const int32_t* t_indptr, const int32_t* t_indices,                \
                               const T* t_data, const double* dw, const int32_t* d_indptr,       \
                               int32_t* d_indices, T* d_data, void* stream);

GSPB200_DECLARE_DIFF_API(f32, float)
GSPB200_DECLARE_DIFF_API(f64, double)

/* ------------------------------------------------------------------ connectivity ---
 * pygsp/graphs/graph.py:192-366, 444-508 on a canonical CSR adjacency W (n x n).  Vertex ids,
 * labels and positions are int32; counters are int64.
 * gsp_cc_labels_*:     the BFS of is_connected (graph.py:343-363, undirected) and of
 *     extract_components (:483-500).  labels[v] = smallest vertex id of v's connected component
 *     (union-find, deterministic).  W must have a symmetric structure; an edge is every stored
 *     entry, or only the entries with weight > 0 when positive_only != 0 (A = W > 0 of
 *     extract_components).  n_components (may be NULL) receives the number of components.
 * gsp_reach_init / gsp_reach_levels: the BFS of is_connected for a directed graph (:343-363),
 *     through W and again through W^T.  visited (n), queue (2 n) and state (4 int64) belong to
 *     the caller.  init marks `source`; each levels call runs BFS levels
 *     [level0, level0 + n_levels) (one launch per level, nothing synchronises).  After levels
 *     [0, L) the search is over when state[L % 3] == 0; state[3] then counts the vertices
 *     reached.
 * gsp_vertex_map:      multiplicity map of a vertex list v (m entries in [0, n), repeats
 *     allowed) -- the row / column selection of W[vertices, :][:, vertices] (:247).
 *     mpos[mptr[u] .. mptr[u + 1]) are the positions p with v[p] == u, increasing; mptr has
 *     n + 1 entries, mpos m.
 * gsp_subgraph_count / gsp_subgraph_fill_*: W[v, :][:, v] (:247) as CSR (m x m).  labels (may be
 *     NULL) keeps an entry (u, c) only when labels[u] == labels[c].  fill writes the entries,
 *     each row in W's column order mapped through mpos: sorted when v is strictly increasing, and
 *     block-diagonal sorted when v lists the vertices by (label, id) and labels is given.
 *     Otherwise the caller sorts the rows (s_rows, may be NULL, receives each entry's row for
 *     gsp_coo_to_csr_*); no two entries coincide.
 * gsp_component_order: the vertices sorted by (label, id) into perm (n); comp_ptr (n + 1) gets
 *     the first position of each component in that order, in increasing order of smallest
 *     vertex, and n at index *n_components (device, may be NULL).
 * gsp_weights_not_one_*: is_weighted (:292), not all(W.data == 1): *flag = 1 if an entry differs
 *     from 1, else 0.
 */
int gsp_reach_init(int64_t n, int32_t source, int32_t* visited, int32_t* queue, int64_t* state,
                   void* stream);
int gsp_reach_levels(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* visited,
                     int32_t* queue, int64_t* state, int64_t level0, int n_levels, void* stream);
int gsp_vertex_map(int64_t n, int64_t m, const int32_t* v, int32_t* mptr, int32_t* mpos,
                   void* stream);
int gsp_subgraph_count(int64_t m, const int32_t* indptr, const int32_t* indices, const int32_t* v,
                       const int32_t* mptr, const int32_t* labels, int32_t* s_indptr,
                       int64_t* nnz, void* stream);
int gsp_component_order(int64_t n, const int32_t* labels, int32_t* perm, int32_t* comp_ptr,
                        int64_t* n_components, void* stream);

#define GSPB200_DECLARE_CONN_API(SUF, T)                                                         \
  int gsp_cc_labels_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,              \
                          const T* data, int positive_only, int32_t* labels,                     \
                          int64_t* n_components, void* stream);                                  \
  int gsp_subgraph_fill_##SUF(int64_t m, const int32_t* indptr, const int32_t* indices,          \
                              const T* data, const int32_t* v, const int32_t* mptr,              \
                              const int32_t* mpos, const int32_t* labels,                        \
                              const int32_t* s_indptr, int32_t* s_indices, T* s_data,            \
                              int32_t* s_rows, void* stream);                                    \
  int gsp_weights_not_one_##SUF(int64_t nnz, const T* data, int32_t* flag, void* stream);

GSPB200_DECLARE_CONN_API(f32, float)
GSPB200_DECLARE_CONN_API(f64, double)

/* ----------------------------------------------------------- multiresolution ---
 * pygsp/reduction.py: Kron reduction, effective resistances and the edge sampler of
 * graph_sparsify (pygsp_b200/reduction.py, csrc/schur.cu).  Kron reduction is always float64.
 * The matrix M (n x n, canonical CSR) is split into kept and removed vertices by `slot`:
 * slot[v] >= 0 for a removed vertex (its position in its component), slot[v] = -1 - (index of v
 * among the kept vertices) for a kept one.  The removed vertices are listed component by
 * component in cvert, component c at cvert[cptr[c] .. cptr[c + 1]); its kept neighbours B, in
 * increasing kept index, at bidx[bptr[c] .. bptr[c + 1]).
 * gsp_schur_small_f64: the blocks -M_BS M_SS^-1 M_SB of linalg.spsolve / dot at reduction.py:358,
 *   one CTA per component listed in comps (n_small entries): Cholesky of M_SS in shared memory,
 *   then |B|^2 COO triplets (row-major over B x B, kept indices) at rows / cols / vals +
 *   out_off[c].  smem_bytes >= 8 (s^2 + s + s b) + 4 b for every listed component.  *status (device)
 *   is set to 1 if some M_SS is not positive definite, else 0.
 * gsp_schur_gather_f64: the dense blocks M_SS (s x s) into A and M_SB (s x nb) into B, both
 *   row-major, of the component whose vertices are cvert[0 .. s) and whose kept neighbours are
 *   bidx[0 .. nb) -- the input of a dense float64 Cholesky for a large component.
 * gsp_edge_resistance_f64: R[e] = Ainv[u][u] + Ainv[v][v] - Ainv[u][v] - Ainv[v][u] for
 *   u = erow[e], v = ecol[e] and a dense row-major Ainv (ld lda) -- the effective resistances
 *   resistance_distances[start_nodes, end_nodes] of graph_sparsify (:84, :101).
 * gsp_sparsify_sample: counts[e] (int64, ne) = how many of q draws from P(e) = weights[e] /
 *   sum(weights) (uint64 integer weights, sum < 2^64) picked e -- dist.rvs(size=q) and the
 *   removed stats.itemfreq of graph_sparsify (:104-115).  Draws come from Philox streams of
 *   `seed` (curand_kernel.h): the counts depend on (seed, weights, q) only.
 * gsp_jl_sketch_f64, gsp_jl_accumulate_f64: the effective resistances of graph_sparsify (:84,
 *   :101) without a dense factor, by the Johnson-Lindenstrauss sketch of Spielman-Srivastava
 *   (csrc/resistance.cu).  L (n x n, canonical float64 CSR, non-positive off-diagonal entries:
 *   only those are read, W = -offdiag(L)), dinv[i] = (W 1)[i]^-1/2 (0 for an isolated vertex),
 *   k columns of which a call handles the block j0 .. j0 + width - 1 (1 <= width <= 256,
 *   j0 + width <= k).
 *   Philox convention: the sign of edge {a < b} in column j is +1 when bit (j mod 128) of the 128
 *   bits of curand4 after curand_init(key, a n + b, 4 (j div 128)) is 0, else -1; bit t of the
 *   128 is bit (t mod 32) of word (t div 32) of (x, y, z, w).
 * gsp_jl_sketch_f64: Y (n x width, row-major, double) := column j - j0 of
 *   D^-1/2 B^T W^1/2 q_j / sqrt(k): Y[i][j - j0] = dinv[i] / sqrt(k) * sum over the off-diagonal
 *   entries (i, v) of row i, in CSR order, of s sqrt(-L_iv) q_j({i, v}), s = +1 when i > v, else
 *   -1.  Every entry of Y is written.
 * gsp_jl_accumulate_f64: R[e] += sum over the block's columns c, in order, of
 *   (dinv[u] U[u][c] - dinv[v] U[v][c])^2 for u = erow[e], v = ecol[e] (ne edges), with U
 *   (n x width, row-major) the solution of D^-1/2 (D - W) D^-1/2 U = Y, D = diag(W 1).
 */
int gsp_schur_small_f64(const int32_t* indptr, const int32_t* indices, const double* data,
                        const int32_t* slot, const int32_t* cvert, const int32_t* cptr,
                        const int32_t* bptr, const int32_t* bidx, int64_t n_small,
                        const int32_t* comps, int smem_bytes, const int64_t* out_off,
                        int32_t* rows, int32_t* cols, double* vals, int32_t* status,
                        void* stream);
int gsp_schur_gather_f64(const int32_t* indptr, const int32_t* indices, const double* data,
                         const int32_t* slot, const int32_t* cvert, int64_t s,
                         const int32_t* bidx, int64_t nb, double* A, double* B, void* stream);
int gsp_edge_resistance_f64(int64_t ne, const int32_t* erow, const int32_t* ecol,
                            const double* ainv, int64_t lda, double* R, void* stream);
int gsp_sparsify_sample(int64_t ne, const uint64_t* weights, int64_t q, uint64_t seed,
                        int64_t* counts, void* stream);
int gsp_jl_sketch_f64(int64_t n, const int32_t* indptr, const int32_t* indices, const double* data,
                      const double* dinv, uint64_t key, int64_t j0, int64_t width, int64_t k,
                      double* Y, void* stream);
int gsp_jl_accumulate_f64(int64_t ne, const int32_t* erow, const int32_t* ecol, const double* U,
                          const double* dinv, int64_t width, double* R, void* stream);
/* Kron reduction by random walks (kron_reduction(method='walks'), csrc/schur_walk.cu): the
 * Schur complement sampler of Durfee, Kyng, Peebles, Rao and Sachdeva.  M (n x n, canonical
 * float64 CSR, symmetric) has weights w_uv = -M_uv (u != v) and excess e_u, an edge to one ground
 * vertex g; slot as above (only its sign is read: < 0 kept, >= 0 removed).
 * gsp_walk_prep_f64: prefix[k] (nnz) := inclusive sum of the weights of row u up to entry k, in
 *   CSR order (the diagonal entry adds 0); total[u] := the row's sum; excess[u] := excess_in[u]
 *   when excess_in is not NULL, else M_uu - total[u]; negative excesses are stored as 0.  *status
 *   (device) gets bit 1 for a positive off-diagonal entry and, without excess_in, bit 2 for an
 *   excess below -1e-12 M_uu.  status is or-ed into, never cleared.
 * gsp_schur_walk_f64: items (edge e) x samples for the n_edges edges (eu[e], ev[e]) of weight
 *   ew[e], item e samples + r, then (ground edge of the removed vertex gu[j]) x samples.  An item
 *   walks from eu (gu) until a kept vertex or g, then from ev until a kept vertex or g, R summing
 *   1/w over the steps of the first walk, then 1/ew[e] (1/excess[gu[j]]), then the second walk's
 *   steps.  Draws: curand_init(key, item, 0); step t of the item (counted over both walks) uses
 *   words 2 (t mod 2) (lo) and 2 (t mod 2) + 1 (hi) of the (t div 2)-th curand4,
 *   U = (((hi << 32) | lo) >> 11) 2^-53, X = U (total[x] + excess[x]): the ground when
 *   X >= total[x] and excess[x] > 0, else the first entry of row x with prefix > X (the last
 *   positive weight when there is none).  With endpoints c1 != c2 (kept indices) and
 *   val = 1 / (R samples), an edge item writes rows / cols / vals[4 item .. 4 item + 4) =
 *   (c1, c2, -val), (c2, c1, -val), (c1, c1, val), (c2, c2, val); with one endpoint g and the
 *   other c, (c, c, val) at 4 item and three empty slots; a ground item writes one slot at
 *   4 n_edges samples + (item - n_edges samples).  An empty slot has row = col = -1.  An item
 *   that needs more than max_steps steps emits nothing and sets bit 4 of *status.  steps (may be
 *   NULL) gets each item's number of steps.  Needs (n_edges + n_ground) samples and
 *   (4 n_edges + n_ground) samples below 2^31.
 */
int gsp_walk_prep_f64(int64_t n, const int32_t* indptr, const int32_t* indices, const double* data,
                      const double* excess_in, double* prefix, double* total, double* excess,
                      int32_t* status, void* stream);
int gsp_schur_walk_f64(const int32_t* indptr, const int32_t* indices, const double* data,
                       const double* prefix, const double* total, const double* excess,
                       const int32_t* slot, int64_t n_edges, const int32_t* eu, const int32_t* ev,
                       const double* ew, int64_t n_ground, const int32_t* gu, int64_t samples,
                       uint64_t key, int64_t max_steps, int32_t* rows, int32_t* cols,
                       double* vals, int32_t* steps, int32_t* status, void* stream);

/* ---------------------------------------------------------------- random graphs ---
 * Draws come from Philox4x32-10 streams of `key` (curand_kernel.h) whose subsequence is a chunk
 * id (SBM) or a slot id (BA): a graph depends on (key, parameters) only, not on the launch
 * shape.  max_blocks caps the grid (0 = the default shape).
 * gsp_sbm_count / gsp_sbm_fill: the pair loop of stochasticblockmodel.py:125-139 (one uniform
 *   per vertex pair) as a Bernoulli process over each block pair's index range, walked by
 *   geometric skips in chunks.  plan (n_blocks x GSPB200_SBM_PLAN_COLS int64, row-major, rows in
 *   increasing cfirst) holds per block pair: n_pairs, chunk length, first global chunk id,
 *   first position of block a and of block b in perm, nb (size of block b; n of the block for
 *   kind 3), kind (0 rectangle, 1 strict lower triangle, 2 lower triangle with the diagonal,
 *   3 n (n - 1) ordered pairs without the diagonal) and mirror (1: an off-diagonal pair also
 *   emits its transpose).  prob (n_blocks x 2 double): p in (0, 1] and log1p(-p).
 *   gsp_sbm_count writes offsets (n_chunks + 1): 0 then the inclusive scan of the entries each
 *   chunk emits.  gsp_sbm_fill writes the COO entries (vertex ids perm[position]) of chunk c at
 *   rows / cols [offsets[c], offsets[c + 1]).
 * gsp_subset_select: a uniform n_s-subset of every pair space s, for Community's exact edge
 *   counts.  The spaces are runs of consecutive plan rows, space s the chunks
 *   [space_chunk_host[s], space_chunk_host[s + 1]) (host, n_spaces + 1, from 0 to n_chunks),
 *   walked by gsp_sbm_count / gsp_sbm_fill with mirror 0, the identity perm and an inflated
 *   probability into the candidates cand_rows / cand_cols (offsets: gsp_sbm_count's).  Each
 *   candidate (u, v) gets the priority (x << 32) | y of the Philox block (u n + v, 2^63) of
 *   `key`; the n_s = target_host[s] lowest (priority, candidate) of each space are kept and
 *   written as (u, v), (v, u) to rows / cols, 2 sum(n_s) entries, space after space.  Synchronises
 *   the stream once; -3 when a space has fewer than n_s candidates (redraw the walk with another
 *   key) or when there are 2^31 candidates or more.
 * gsp_barabasi_albert: the attachment loop of barabasialbert.py:54-64.  Writes 2 m (n - m0)
 *   COO entries, (i, v) and (v, i) for each of the m targets v of each vertex i >= m0, in
 *   rounds of one launch each (the call synchronises the stream every few rounds);
 *   *rounds_host_out gets the number of rounds.  -3 if the rounds do not finish.
 */
#define GSPB200_SBM_PLAN_COLS 8
int gsp_sbm_count(int64_t n_chunks, int64_t n_blocks, const int64_t* plan, const double* prob,
                  uint64_t key, int64_t* offsets, int max_blocks, void* stream);
int gsp_sbm_fill(int64_t n_chunks, int64_t n_blocks, const int64_t* plan, const double* prob,
                 uint64_t key, const int32_t* perm, const int64_t* offsets, int32_t* rows,
                 int32_t* cols, int max_blocks, void* stream);
int gsp_subset_select(int64_t n, int64_t n_chunks, const int64_t* offsets, int64_t n_spaces,
                      const int64_t* space_chunk_host, const int64_t* target_host, uint64_t key,
                      const int32_t* cand_rows, const int32_t* cand_cols, int32_t* rows,
                      int32_t* cols, int max_blocks, void* stream);
int gsp_barabasi_albert(int64_t n, int64_t m0, int64_t m, uint64_t key, int32_t* rows,
                        int32_t* cols, int max_blocks, int* rounds_host_out, void* stream);

/* ---------------------------------------------------------------- random regular ---
 * gsp_random_regular: a simple undirected k-regular graph on n vertices (randomregular.py) by
 *   stub pairing; n k even, 0 <= k < n (or k = 0), n k < 2^31, max_iter >= 1 attempts.  Every draw
 *   is Philox4x32-10 of `key` at subsequence (attempt << 32) | phase (phase r: bulk round r;
 *   GSPB200_RR_TAIL_STREAM, GSPB200_RR_SWITCH_STREAM) and an offset that is a pool position or a
 *   draw number, so the graph depends on (key, n, k, max_iter) only, not on max_blocks (which caps
 *   the grid; 0 = the default shape).  While the pool holds more than GSPB200_RR_TAIL_STUBS stubs,
 *   rounds pair it after a stable sort by priority; one CTA finishes it by the reference's
 *   sequential rule, restarting the attempt on a stuck pool (an exact check after
 *   GSPB200_RR_CHECK_AFTER rejections in a row) or after GSPB200_RR_TAIL_DRAWS draws; the last
 *   attempt places the remaining stubs by edge switches instead (at most GSPB200_RR_SWITCH_DRAWS
 *   draws per stub pair, else the partial graph is kept).  Writes (u, v), (v, u) per edge to
 *   rows / cols (room for n k entries); *entries_host_out gets their number (n k unless the graph
 *   is partial), *attempts_host_out the attempts used, *rounds_host_out the rounds of all
 *   attempts.  Synchronises the stream once per round and per attempt.  -3 if an attempt's rounds
 *   do not reach the tail within GSPB200_RR_MAX_ROUNDS rounds.
 * gsp_random_regular_complement: the complement (every j != i that is not a neighbour) of the
 *   canonical CSR indptr / indices (n x n, symmetric, no loops), written as canonical CSR:
 *   out_indptr (n + 1) and out_indices (nnz = n (n - 1) - indptr[n], given by the caller).
 */
#define GSPB200_RR_TAIL_STUBS 4096
#define GSPB200_RR_CHECK_AFTER 32
#define GSPB200_RR_TAIL_DRAWS (1 << 22)
#define GSPB200_RR_SWITCH_DRAWS (1 << 16)
#define GSPB200_RR_MAX_ROUNDS 4096
#define GSPB200_RR_TAIL_STREAM 0xFFFFFFFFull
#define GSPB200_RR_SWITCH_STREAM 0xFFFFFFFEull
int gsp_random_regular(int64_t n, int64_t k, int max_iter, uint64_t key, int32_t* rows,
                       int32_t* cols, int max_blocks, int* attempts_host_out,
                       int* rounds_host_out, int64_t* entries_host_out, void* stream);
int gsp_random_regular_complement(int64_t n, int64_t nnz, const int32_t* indptr,
                                  const int32_t* indices, int32_t* out_indptr,
                                  int32_t* out_indices, void* stream);

/* ------------------------------------------------------------- structured graphs ---
 * The closed-form models of pygsp/graphs/{path,comet,star,torus,fullconnected,randomring}.py as
 * canonical CSR: each count writes indptr (n + 1) and the total, each fill the rows.
 * gsp_comet_*: star 0 - 1..k and tail path k - ... - n-1 (comet.py); k = 0 is the path graph
 *   (path.py), k = n - 1 the star (star.py); directed != 0 (k = 0 only): edges i -> i+1.  Unit
 *   weights.
 * gsp_torus_*: torus.py, n = nv mv vertices v = i nv + t with neighbours t +- 1 (mod nv) and
 *   i +- 1 (mod mv); coinciding neighbours are one entry whose weight counts them (2 when
 *   nv <= 2 or mv <= 2, self-loops when nv = 1 or mv = 1), as the reference sums its duplicates.
 * gsp_full_connected_indptr / _fill_*: fullconnected.py, every j != i with weight 1;
 *   n (n - 1) < 2^31.  The indptr call is the count; *nnz is n (n - 1).
 * gsp_random_ring_count / _fill_*: randomring.py on sorted angles (n >= 3, double): the edge
 *   i - i+1 and the closing edge 0 - n-1 have weight width / (angle difference), the closing
 *   difference (2 pi + a[0]) - a[n - 1]; double, rounded once.  Zero differences are not stored.
 * gsp_low_stretch_tree_coo: the 2 4^levels - 2 COO triplets of lowstretchtree.py (levels = k),
 *   in the reference's order, for gsp_coo_to_csr_* with unit values.  levels in 1..15.
 * gsp_line_graph_count / _fill_*: linegraph.py, (D != 0)^T (D != 0) - I (n_edges x n_edges) from
 *   the edge list (sources, targets; gsp_edge_list_*) and D's indptr / indices
 *   (gsp_incidence_fill_*).  w_indptr / w_indices is W, searched for the reciprocal edge t -> s
 *   when directed != 0.  fill writes each row sorted: value 1 for every edge sharing an end with
 *   edge k, or the single entry (k, k) = -1 for a self-loop.
 */
int gsp_comet_count(int64_t n, int64_t k, int directed, int32_t* indptr, int64_t* nnz,
                    void* stream);
int gsp_torus_count(int64_t nv, int64_t mv, int32_t* indptr, int64_t* nnz, void* stream);
int gsp_full_connected_indptr(int64_t n, int32_t* indptr, int64_t* nnz, void* stream);
int gsp_random_ring_count(int64_t n, const double* angles, int32_t* indptr, int64_t* nnz,
                          void* stream);
int gsp_low_stretch_tree_coo(int levels, int32_t* rows, int32_t* cols, void* stream);
int gsp_line_graph_count(int64_t n_edges, const int32_t* sources, const int32_t* targets,
                         const int32_t* d_indptr, const int32_t* w_indptr,
                         const int32_t* w_indices, int directed, int32_t* lg_indptr, int64_t* nnz,
                         void* stream);

#define GSPB200_DECLARE_STRUCT_API(SUF, T)                                                       \
  int gsp_comet_fill_##SUF(int64_t n, int64_t k, int directed, const int32_t* indptr,            \
                           int32_t* indices, T* data, void* stream);                             \
  int gsp_torus_fill_##SUF(int64_t nv, int64_t mv, const int32_t* indptr, int32_t* indices,      \
                           T* data, void* stream);                                               \
  int gsp_full_connected_fill_##SUF(int64_t n, int32_t* indices, T* data, void* stream);         \
  int gsp_random_ring_fill_##SUF(int64_t n, const double* angles, double width,                  \
                                 const int32_t* indptr, int32_t* indices, T* data,               \
                                 void* stream);                                                  \
  int gsp_line_graph_fill_##SUF(int64_t n_edges, const int32_t* sources, const int32_t* targets,  \
                                const int32_t* d_indptr, const int32_t* d_indices,               \
                                const int32_t* w_indptr, const int32_t* w_indices, int directed, \
                                const int32_t* lg_indptr, int32_t* lg_indices, T* lg_data,       \
                                void* stream);

GSPB200_DECLARE_STRUCT_API(f32, float)
GSPB200_DECLARE_STRUCT_API(f64, double)

/* ------------------------------------------------------------ tree multiresolution ---
 * pygsp/reduction.py: tree_multiresolution (pygsp_b200/reduction.py, csrc/tree.cu).  The tree is
 * the canonical symmetric CSR indptr / indices / data (n x n, 1 <= n <= 2^30, nnz stored entries);
 * diagonal entries are ignored.  Vertex ids are int32.
 * gsp_tree_arc_count: arc_ptr (n + 1) := 0 and the inclusive scan of each row's off-diagonal
 *   entries (the arcs, in CSR order); *n_arcs (device, int64) := their number.
 * gsp_tree_root_*: depth, parent (int32, n) and wpar (double, n: the weight of the edge to the
 *   parent, as stored, widened) of every vertex from `root`; depth[root] = 0, parent[root] = root,
 *   wpar[root] = 0.  Needs a connected graph with n_arcs = 2 (n - 1) (a tree) and arc_ptr from
 *   gsp_tree_arc_count.  Euler tour (twin by binary search, successor the next arc of the twin's
 *   row) ranked by ceil(log2 n_arcs) rounds of pointer jumping, then a scan of +-1 over the tour:
 *   O(log n) launches, no host synchronisation.
 * gsp_tree_keep: new_id (n + 1) := 0 and the inclusive scan of (depth[v] even), i.e. new_id[v] is
 *   v's id among the kept (even-depth) vertices; *n_new (device, int64) := their number.
 * gsp_tree_coarsen_*: one level.  Every kept v (new id i) writes keep[i] = v (int64) and
 *   new_depth[i] = depth[v] / 2; the root new_parent[i] = i, new_wpar[i] = 0; any other kept v, with
 *   p = parent[v], g = parent[p] and j = new_id[g], new_parent[i] = j and the edge (i, j) of weight
 *   c = (T) combine(wpar[v], wpar[p]), in double, for method GSPB200_TREE_UNWEIGHTED (1),
 *   GSPB200_TREE_SUM (wv + wp) or GSPB200_TREE_RESISTANCE (1 / (1 / wv + 1 / wp)); new_wpar[i] = c
 *   widened.  The edges are written as COO at rows / cols / vals [e] = (i, j, c) and [m + e] =
 *   (j, i, c), m = n_new - 1, e the edge's place among the kept non-root vertices.
 */
#define GSPB200_TREE_UNWEIGHTED 0
#define GSPB200_TREE_SUM 1
#define GSPB200_TREE_RESISTANCE 2
int gsp_tree_arc_count(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* arc_ptr,
                       int64_t* n_arcs, void* stream);
int gsp_tree_keep(int64_t n, const int32_t* depth, int32_t* new_id, int64_t* n_new,
                  void* stream);

#define GSPB200_DECLARE_TREE_API(SUF, T)                                                         \
  int gsp_tree_root_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,  \
                          const T* data, const int32_t* arc_ptr, int32_t root, int32_t* depth,   \
                          int32_t* parent, double* wpar, void* stream);                          \
  int gsp_tree_coarsen_##SUF(int64_t n, int64_t n_new, const int32_t* depth,                      \
                             const int32_t* parent, const double* wpar, const int32_t* new_id,   \
                             int32_t root, int method, int64_t* keep, int32_t* rows,             \
                             int32_t* cols, T* vals, int32_t* new_depth, int32_t* new_parent,    \
                             double* new_wpar, void* stream);

GSPB200_DECLARE_TREE_API(f32, float)
GSPB200_DECLARE_TREE_API(f64, double)

#ifdef __cplusplus
}
#endif
#endif /* GSPB200_H_ */
