// Structured graph models and the line graph, built in HBM.
//
// Replaces the host COO assembly of the reference's path.py, comet.py, star.py, torus.py,
// fullconnected.py, randomring.py, lowstretchtree.py and linegraph.py:
//   * Path / Comet / Star, Torus, FullConnected and RandomRing: every row has a closed form, so
//     count -> scan_rows -> fill writes canonical CSR (sorted, unique columns) directly, as the
//     Grid2d kernels do: no COO, no sort.
//   * LowStretchTree: the reference's COO triplets, each decoded from its position in the
//     recursive concatenation of lowstretchtree.py; gsp_coo_to_csr_* assembles them.
//   * LineGraph: W = (D != 0)^T (D != 0) - I of linegraph.py, from the edge list and the rows of
//     D (row v lists the edges incident to v in increasing edge id, csrc/difference.cu).  Row k
//     of edge (s, t) is the sorted union of D_s and D_t without k: one warp per row merges the
//     two lists in 32-wide windows of the merge, each lane finding its element on the merge-path
//     diagonal, so that the stores of a window are contiguous.
#include "common.cuh"
#include "gspb200.h"

namespace gsp {

constexpr int kStructThreads = 256;
constexpr double kTwoPi = 2.0 * 3.141592653589793;   // 2 * np.pi, exactly

static inline int struct_blocks(int64_t n) {
  return (int)ceil_div(n > 0 ? n : 1, kStructThreads);
}

// ------------------------------------------------------------- Path / Comet / Star ---
// Star 0 - 1..k, tail path k - k+1 - ... - n-1 (k = 0: the path graph).  Directed (k = 0 only):
// i -> i+1.  Row 0 of a star (k >= 1) holds 1..k; every other row at most two columns, written
// by comet_row in increasing order.
__device__ __forceinline__ int comet_row(int64_t n, int64_t k, int directed, int64_t i,
                                         int64_t* c) {
  int m = 0;
  if (directed) {
    if (i + 1 < n) c[m++] = i + 1;
    return m;
  }
  if (i >= 1 && i <= k) c[m++] = 0;              // star branch
  if (i >= k) {                                  // tail
    if (i - 1 >= k) c[m++] = i - 1;
    if (i + 1 < n) c[m++] = i + 1;
  }
  return m;
}

__global__ void comet_count_kernel(int64_t n, int64_t k, int directed, int32_t* indptr) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i == 0) indptr[0] = 0;
  if (i >= n) return;
  int64_t c[2];
  indptr[i + 1] = (i == 0 && k >= 1) ? (int32_t)k : comet_row(n, k, directed, i, c);
}

// one thread per row and, for i < k, per entry of the hub row 0 (which starts at 0)
template <typename T>
__global__ void comet_fill_kernel(int64_t n, int64_t k, int directed,
                                  const int32_t* __restrict__ indptr, int32_t* indices, T* data) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < k) {
    indices[i] = (int32_t)(i + 1);
    data[i] = T(1);
  }
  if (i >= n || (i == 0 && k >= 1)) return;
  int64_t c[2];
  const int m = comet_row(n, k, directed, i, c);
  const int o = __ldg(indptr + i);
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (j < m) {
      indices[o + j] = (int32_t)c[j];
      data[o + j] = T(1);
    }
  }
}

// ------------------------------------------------------------------------- Torus ---
// Vertex v = i * nv + t (ring i < mv, position t < nv) has the four neighbours t +- 1 (mod nv)
// in its ring and i +- 1 (mod mv) across rings, each of weight 1.  Coinciding neighbours are
// merged and their weights added, which is the reference's sum of duplicate COO entries
// (nv <= 2 or mv <= 2: weight 2; nv = 1 or mv = 1: self-loops).
// the four candidates of row v, sorted
__device__ __forceinline__ void torus_candidates(int64_t nv, int64_t mv, int64_t v, int64_t* c) {
  const int64_t i = v / nv, t = v - i * nv;
  c[0] = i * nv + (t + 1) % nv;
  c[1] = i * nv + (t + nv - 1) % nv;
  c[2] = ((i + 1) % mv) * nv + t;
  c[3] = ((i + mv - 1) % mv) * nv + t;
  auto cswap = [&](int a, int b) {
    if (c[a] > c[b]) { const int64_t x = c[a]; c[a] = c[b]; c[b] = x; }
  };
  cswap(0, 1); cswap(2, 3); cswap(0, 2); cswap(1, 3); cswap(1, 2);
}

__global__ void torus_count_kernel(int64_t nv, int64_t mv, int32_t* indptr) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v == 0) indptr[0] = 0;
  if (v >= nv * mv) return;
  int64_t c[4];
  torus_candidates(nv, mv, v, c);
  indptr[v + 1] = 1 + int(c[1] != c[0]) + int(c[2] != c[1]) + int(c[3] != c[2]);
}

template <typename T>
__global__ void torus_fill_kernel(int64_t nv, int64_t mv, const int32_t* __restrict__ indptr,
                                  int32_t* indices, T* data) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= nv * mv) return;
  int64_t c[4];
  torus_candidates(nv, mv, v, c);
  int o = __ldg(indptr + v);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (j > 0 && c[j] == c[j - 1]) continue;     // counted with the first of its run
    int w = 1;
#pragma unroll
    for (int l = j + 1; l < 4; ++l) w += int(c[l] == c[j]);
    indices[o] = (int32_t)c[j];
    data[o++] = T(w);
  }
}

// ----------------------------------------------------------------- FullConnected ---
// Row i holds every j != i: entry e = i (n - 1) + r has column r + (r >= i).  The caller
// guarantees n (n - 1) < 2^31.
__global__ void full_connected_indptr_kernel(int64_t n, int32_t* indptr, int64_t* nnz) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i == 0 && nnz) *nnz = n * (n - 1);
  if (i <= n) indptr[i] = (int32_t)(i * (n - 1));
}

template <typename T>
__global__ void full_connected_fill_kernel(uint32_t n, uint32_t nnz, int32_t* indices, T* data) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= nnz) return;
  const uint32_t row = e / (n - 1), r = e - row * (n - 1);
  indices[e] = (int32_t)(r + (r >= row));
  data[e] = T(1);
}

// -------------------------------------------------------------------- RandomRing ---
// Sorted angles a (n >= 3).  Edge j joins j and j + 1 for j < n - 1, with angle difference
// a[j + 1] - a[j]; edge n - 1 closes the ring between 0 and n - 1 with (2 pi + a[0]) - a[n - 1].
// Weight width / difference in double, rounded once to T.  An edge of difference 0 is not
// stored: the reference's symmetrisation drops the zero before inverting the weights.
__device__ __forceinline__ double ring_gap(int64_t n, const double* __restrict__ a, int64_t j) {
  return j < n - 1 ? __ldg(a + j + 1) - __ldg(a + j) : (kTwoPi + __ldg(a)) - __ldg(a + n - 1);
}

// row i: (column, edge) pairs in increasing column order
__device__ __forceinline__ void ring_row(int64_t n, int64_t i, int64_t* col, int64_t* edge) {
  if (i == 0) {
    col[0] = 1; edge[0] = 0; col[1] = n - 1; edge[1] = n - 1;
  } else if (i == n - 1) {
    col[0] = 0; edge[0] = n - 1; col[1] = n - 2; edge[1] = n - 2;
  } else {
    col[0] = i - 1; edge[0] = i - 1; col[1] = i + 1; edge[1] = i;
  }
}

__global__ void random_ring_count_kernel(int64_t n, const double* __restrict__ angles,
                                         int32_t* indptr) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i == 0) indptr[0] = 0;
  if (i >= n) return;
  int64_t col[2], edge[2];
  ring_row(n, i, col, edge);
  indptr[i + 1] = int(ring_gap(n, angles, edge[0]) != 0) + int(ring_gap(n, angles, edge[1]) != 0);
}

template <typename T>
__global__ void random_ring_fill_kernel(int64_t n, const double* __restrict__ angles, double width,
                                        const int32_t* __restrict__ indptr, int32_t* indices,
                                        T* data) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t col[2], edge[2];
  ring_row(n, i, col, edge);
  int o = __ldg(indptr + i);
  for (int j = 0; j < 2; ++j) {
    const double gap = ring_gap(n, angles, edge[j]);
    if (gap == 0) continue;
    indices[o] = (int32_t)col[j];
    data[o++] = T(width / gap);
  }
}

// ---------------------------------------------------------------- LowStretchTree ---
// lowstretchtree.py builds its triplets level by level: level 0 is the six entries of the 2 x 2
// block; level p >= 1 is four copies of level p - 1, shifted by c 4^p (c = 0..3), followed by
// six connector entries.  Level p holds S_p = 2 4^(p+1) - 2 entries.  Entry e of the top level
// is decoded from the top down: the copy it falls in adds c 4^p to both ends, and either a
// connector or the base block ends the descent.
__device__ __forceinline__ void lst_entry(int levels, int64_t e, int64_t* row, int64_t* col) {
  const int base_i[6] = {0, 0, 1, 2, 2, 3};
  const int base_j[6] = {1, 2, 1, 3, 0, 2};
  int64_t offset = 0;
  for (int p = levels - 1; p >= 1; --p) {
    const int64_t q = int64_t(1) << (2 * p);   // 4^p
    const int64_t sub = 2 * q - 2;             // S_{p-1}
    if (e < 4 * sub) {
      const int64_t c = e / sub;
      e -= c * sub;
      offset += c * q;
      continue;
    }
    const int64_t a = q - 1, b = (5 * q + 1) / 3 - 1, m = q + (4 * q + 2) / 3 - 1, d = 3 * q;
    const int64_t ii[6] = {a, a, m, b, m, d};
    const int64_t jj[6] = {b, m, d, a, a, m};
    *row = offset + ii[e - 4 * sub];
    *col = offset + jj[e - 4 * sub];
    return;
  }
  *row = offset + base_i[e];
  *col = offset + base_j[e];
}

__global__ void low_stretch_tree_kernel(int levels, int64_t nnz, int32_t* rows, int32_t* cols) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= nnz) return;
  int64_t r, c;
  lst_entry(levels, e, &r, &c);
  rows[e] = (int32_t)r;
  cols[e] = (int32_t)c;
}

// --------------------------------------------------------------------- LineGraph ---
// Edge k = (s, t).  D_s and D_t both hold k, and both hold the reciprocal edge k' = (t, s) when
// the graph is directed and W stores it; no other edge has both ends in {s, t}.  So row k has
// |D_s| + |D_t| - 2 - [k' exists] entries.  A loop edge has an empty column of D: its row is
// the single entry (k, k) = -1 of "- I".

// first position in [lo, hi) whose value is >= key
__device__ __forceinline__ int lower_bound_idx(const int32_t* __restrict__ v, int lo, int hi,
                                               int key) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(v + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// edge id of t -> s in a directed graph (its position in W), or -1
__device__ __forceinline__ int reciprocal_edge(const int32_t* __restrict__ w_indptr,
                                               const int32_t* __restrict__ w_indices, int s,
                                               int t) {
  const int end = __ldg(w_indptr + t + 1);
  const int p = lower_bound_idx(w_indices, __ldg(w_indptr + t), end, s);
  return p < end && __ldg(w_indices + p) == s ? p : -1;
}

__global__ void line_graph_count_kernel(int64_t ne, const int32_t* __restrict__ sources,
                                        const int32_t* __restrict__ targets,
                                        const int32_t* __restrict__ d_indptr,
                                        const int32_t* __restrict__ w_indptr,
                                        const int32_t* __restrict__ w_indices, int directed,
                                        int32_t* lg_indptr) {
  const int64_t k = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (k == 0) lg_indptr[0] = 0;
  if (k >= ne) return;
  const int s = __ldg(sources + k), t = __ldg(targets + k);
  int c = 1;
  if (s != t) {                 // |D_s| + |D_t| <= nnz(D) < 2^31
    c = (__ldg(d_indptr + s + 1) - __ldg(d_indptr + s)) +
        (__ldg(d_indptr + t + 1) - __ldg(d_indptr + t)) - 2;
    if (directed && reciprocal_edge(w_indptr, w_indices, s, t) >= 0) --c;
  }
  lg_indptr[k + 1] = c;
}

// One warp per row.  The merge of A = D_s and B = D_t (A first on ties) is cut into windows of
// 32 positions; lane l takes position base + l, finds how many of A precede it by binary search
// on the merge-path diagonal, and keeps its element unless it is k (twice in the merge) or B's
// copy of k'.  A ballot compacts the kept elements of the window into contiguous slots.
template <typename T>
__global__ void __launch_bounds__(kStructThreads)
line_graph_fill_kernel(int64_t ne, const int32_t* __restrict__ sources,
                       const int32_t* __restrict__ targets, const int32_t* __restrict__ d_indptr,
                       const int32_t* __restrict__ d_indices, const int32_t* __restrict__ w_indptr,
                       const int32_t* __restrict__ w_indices, int directed,
                       const int32_t* __restrict__ lg_indptr, int32_t* lg_indices, T* lg_data) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  for (int64_t k = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; k < ne; k += warps) {
    const int s = __ldg(sources + k), t = __ldg(targets + k);
    int out = __ldg(lg_indptr + k);
    if (s == t) {
      if (lane == 0) {
        lg_indices[out] = (int32_t)k;
        lg_data[out] = T(-1);
      }
      continue;
    }
    const int a0 = __ldg(d_indptr + s), b0 = __ldg(d_indptr + t);
    const int a = __ldg(d_indptr + s + 1) - a0, b = __ldg(d_indptr + t + 1) - b0;
    const int32_t* A = d_indices + a0;
    const int32_t* B = d_indices + b0;
    const int kp = directed ? reciprocal_edge(w_indptr, w_indices, s, t) : -1;
    for (int base = 0; base < a + b; base += 32) {
      const int p = base + lane;
      int v = 0;
      bool keep = false;
      if (p < a + b) {
        int lo = max(0, p - b), hi = min(p, a);
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (__ldg(A + mid) <= __ldg(B + p - 1 - mid)) lo = mid + 1; else hi = mid;
        }
        const int i = lo, j = p - lo;
        const bool from_a = i < a && (j >= b || __ldg(A + i) <= __ldg(B + j));
        v = from_a ? __ldg(A + i) : __ldg(B + j);
        keep = v != k && !(!from_a && v == kp);
      }
      const unsigned mask = __ballot_sync(0xffffffffu, keep);
      if (keep) {
        const int o = out + __popc(mask & ((1u << lane) - 1u));
        lg_indices[o] = v;
        lg_data[o] = T(1);
      }
      out += __popc(mask);
    }
  }
}

// ------------------------------------------------------------------ drivers ------
int comet_count(int64_t n, int64_t k, int directed, int32_t* indptr, int64_t* nnz,
                cudaStream_t st) {
  comet_count_kernel<<<struct_blocks(n), kStructThreads, 0, st>>>(n, k, directed, indptr);
  GSP_LAUNCH_CHECK("comet_count");
  return scan_rows(indptr, n, nnz, st);
}

template <typename T>
int comet_fill(int64_t n, int64_t k, int directed, const int32_t* indptr, int32_t* indices,
               T* data, cudaStream_t st) {
  if (n == 0) return GSP_OK;
  comet_fill_kernel<T><<<struct_blocks(std::max(n, k)), kStructThreads, 0, st>>>(
      n, k, directed, indptr, indices, data);
  GSP_LAUNCH_CHECK("comet_fill");
  return GSP_OK;
}

int torus_count(int64_t nv, int64_t mv, int32_t* indptr, int64_t* nnz, cudaStream_t st) {
  torus_count_kernel<<<struct_blocks(nv * mv), kStructThreads, 0, st>>>(nv, mv, indptr);
  GSP_LAUNCH_CHECK("torus_count");
  return scan_rows(indptr, nv * mv, nnz, st);
}

template <typename T>
int torus_fill(int64_t nv, int64_t mv, const int32_t* indptr, int32_t* indices, T* data,
               cudaStream_t st) {
  if (nv * mv == 0) return GSP_OK;
  torus_fill_kernel<T><<<struct_blocks(nv * mv), kStructThreads, 0, st>>>(nv, mv, indptr,
                                                                          indices, data);
  GSP_LAUNCH_CHECK("torus_fill");
  return GSP_OK;
}

int full_connected_indptr(int64_t n, int32_t* indptr, int64_t* nnz, cudaStream_t st) {
  full_connected_indptr_kernel<<<struct_blocks(n + 1), kStructThreads, 0, st>>>(n, indptr, nnz);
  GSP_LAUNCH_CHECK("full_connected_indptr");
  return GSP_OK;
}

template <typename T>
int full_connected_fill(int64_t n, int32_t* indices, T* data, cudaStream_t st) {
  const int64_t nnz = n * (n - 1);
  if (nnz <= 0) return GSP_OK;
  full_connected_fill_kernel<T><<<struct_blocks(nnz), kStructThreads, 0, st>>>(
      (uint32_t)n, (uint32_t)nnz, indices, data);
  GSP_LAUNCH_CHECK("full_connected_fill");
  return GSP_OK;
}

int random_ring_count(int64_t n, const double* angles, int32_t* indptr, int64_t* nnz,
                      cudaStream_t st) {
  random_ring_count_kernel<<<struct_blocks(n), kStructThreads, 0, st>>>(n, angles, indptr);
  GSP_LAUNCH_CHECK("random_ring_count");
  return scan_rows(indptr, n, nnz, st);
}

template <typename T>
int random_ring_fill(int64_t n, const double* angles, double width, const int32_t* indptr,
                     int32_t* indices, T* data, cudaStream_t st) {
  random_ring_fill_kernel<T><<<struct_blocks(n), kStructThreads, 0, st>>>(n, angles, width,
                                                                          indptr, indices, data);
  GSP_LAUNCH_CHECK("random_ring_fill");
  return GSP_OK;
}

int low_stretch_tree_coo(int levels, int32_t* rows, int32_t* cols, cudaStream_t st) {
  const int64_t nnz = 2 * (int64_t(1) << (2 * levels)) - 2;
  low_stretch_tree_kernel<<<struct_blocks(nnz), kStructThreads, 0, st>>>(levels, nnz, rows, cols);
  GSP_LAUNCH_CHECK("low_stretch_tree");
  return GSP_OK;
}

int line_graph_count(int64_t ne, const int32_t* sources, const int32_t* targets,
                     const int32_t* d_indptr, const int32_t* w_indptr, const int32_t* w_indices,
                     int directed, int32_t* lg_indptr, int64_t* nnz, cudaStream_t st) {
  line_graph_count_kernel<<<struct_blocks(ne), kStructThreads, 0, st>>>(
      ne, sources, targets, d_indptr, w_indptr, w_indices, directed, lg_indptr);
  GSP_LAUNCH_CHECK("line_graph_count");
  return scan_rows(lg_indptr, ne, nnz, st);
}

template <typename T>
int line_graph_fill(int64_t ne, const int32_t* sources, const int32_t* targets,
                    const int32_t* d_indptr, const int32_t* d_indices, const int32_t* w_indptr,
                    const int32_t* w_indices, int directed, const int32_t* lg_indptr,
                    int32_t* lg_indices, T* lg_data, cudaStream_t st) {
  if (ne == 0) return GSP_OK;
  constexpr int warps_per_block = kStructThreads / 32;
  // one resident wave; every warp then walks rows with a stride of the whole grid
  const int64_t blocks = std::min<int64_t>(ceil_div(ne, warps_per_block),
                                           int64_t(sm_count()) * (2048 / kStructThreads));
  line_graph_fill_kernel<T><<<(int)blocks, kStructThreads, 0, st>>>(
      ne, sources, targets, d_indptr, d_indices, w_indptr, w_indices, directed, lg_indptr,
      lg_indices, lg_data);
  GSP_LAUNCH_CHECK("line_graph_fill");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
#define GSP_STRUCT_API(SUF, T)                                                                  \
  int gsp_comet_fill_##SUF(int64_t n, int64_t k, int directed, const int32_t* indptr,           \
                           int32_t* indices, T* data, void* stream) {                           \
    GSP_REQUIRE(n >= 0 && k >= 0 && (k == 0 || (k < n && !directed)), "bad comet shape");       \
    return gsp::comet_fill<T>(n, k, directed, indptr, indices, data, gsp::as_stream(stream));  \
  }                                                                                             \
  int gsp_torus_fill_##SUF(int64_t nv, int64_t mv, const int32_t* indptr, int32_t* indices,     \
                           T* data, void* stream) {                                             \
    GSP_REQUIRE(nv >= 1 && mv >= 1 && nv * mv < (int64_t(1) << 31), "bad torus shape");         \
    return gsp::torus_fill<T>(nv, mv, indptr, indices, data, gsp::as_stream(stream));           \
  }                                                                                             \
  int gsp_full_connected_fill_##SUF(int64_t n, int32_t* indices, T* data, void* stream) {       \
    GSP_REQUIRE(n >= 0 && n * (n - 1) < (int64_t(1) << 31), "n (n - 1) must be < 2^31");        \
    return gsp::full_connected_fill<T>(n, indices, data, gsp::as_stream(stream));               \
  }                                                                                             \
  int gsp_random_ring_fill_##SUF(int64_t n, const double* angles, double width,                 \
                                 const int32_t* indptr, int32_t* indices, T* data,              \
                                 void* stream) {                                                \
    GSP_REQUIRE(n >= 3 && n < (int64_t(1) << 30), "bad ring size");                             \
    return gsp::random_ring_fill<T>(n, angles, width, indptr, indices, data,                    \
                                    gsp::as_stream(stream));                                    \
  }                                                                                             \
  int gsp_line_graph_fill_##SUF(int64_t n_edges, const int32_t* sources, const int32_t* targets, \
                                const int32_t* d_indptr, const int32_t* d_indices,              \
                                const int32_t* w_indptr, const int32_t* w_indices, int directed, \
                                const int32_t* lg_indptr, int32_t* lg_indices, T* lg_data,      \
                                void* stream) {                                                 \
    GSP_REQUIRE(n_edges >= 0 && n_edges < (int64_t(1) << 31), "n_edges out of range");         \
    return gsp::line_graph_fill<T>(n_edges, sources, targets, d_indptr, d_indices, w_indptr,    \
                                   w_indices, directed, lg_indptr, lg_indices, lg_data,         \
                                   gsp::as_stream(stream));                                     \
  }

extern "C" {
int gsp_comet_count(int64_t n, int64_t k, int directed, int32_t* indptr, int64_t* nnz,
                    void* stream) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31) && k >= 0 && (k == 0 || (k < n && !directed)),
              "bad comet shape");
  return gsp::comet_count(n, k, directed, indptr, nnz, gsp::as_stream(stream));
}
int gsp_torus_count(int64_t nv, int64_t mv, int32_t* indptr, int64_t* nnz, void* stream) {
  GSP_REQUIRE(nv >= 1 && mv >= 1 && nv * mv < (int64_t(1) << 31), "bad torus shape");
  return gsp::torus_count(nv, mv, indptr, nnz, gsp::as_stream(stream));
}
int gsp_full_connected_indptr(int64_t n, int32_t* indptr, int64_t* nnz, void* stream) {
  GSP_REQUIRE(n >= 0 && n * (n - 1) < (int64_t(1) << 31), "n (n - 1) must be < 2^31");
  return gsp::full_connected_indptr(n, indptr, nnz, gsp::as_stream(stream));
}
int gsp_random_ring_count(int64_t n, const double* angles, int32_t* indptr, int64_t* nnz,
                          void* stream) {
  GSP_REQUIRE(n >= 3 && n < (int64_t(1) << 30), "bad ring size");
  return gsp::random_ring_count(n, angles, indptr, nnz, gsp::as_stream(stream));
}
int gsp_low_stretch_tree_coo(int levels, int32_t* rows, int32_t* cols, void* stream) {
  GSP_REQUIRE(levels >= 1 && levels <= 15, "levels must be in 1..15");
  return gsp::low_stretch_tree_coo(levels, rows, cols, gsp::as_stream(stream));
}
int gsp_line_graph_count(int64_t n_edges, const int32_t* sources, const int32_t* targets,
                         const int32_t* d_indptr, const int32_t* w_indptr,
                         const int32_t* w_indices, int directed, int32_t* lg_indptr, int64_t* nnz,
                         void* stream) {
  GSP_REQUIRE(n_edges >= 0 && n_edges < (int64_t(1) << 31), "n_edges out of range");
  return gsp::line_graph_count(n_edges, sources, targets, d_indptr, w_indptr, w_indices, directed,
                               lg_indptr, nnz, gsp::as_stream(stream));
}
GSP_STRUCT_API(f32, float)
GSP_STRUCT_API(f64, double)
}
