// Graph differential operator: edge list, incidence matrix D (N x Ne) and its transpose,
// built in HBM from the adjacency.
//
// Replaces, for pygsp/graphs/difference.py:144-166 and graph.py:1019-1029:
//   * sparse.triu(W, format='coo') / W.tocoo()                  (graph.py:1019-1026)
//   * the COO -> csc_matrix assembly of D and eliminate_zeros()   (difference.py:147-166)
// Everything is count -> scan -> fill on canonical CSR (sorted, unique columns); no sort, no
// atomics, no host copy.
//
// Edges are numbered in row-major CSR order: the entries of W with col >= row for an
// undirected graph (self-loops included), every stored entry for a directed one (the edge
// offsets are then W's indptr).  Column k of D -- row k of D^T -- holds -v_s at the source and
// +v_t at the target, in increasing vertex order, or nothing for a self-loop (the reference's
// two entries of a loop cancel and eliminate_zeros() drops them):
//   combinatorial  v = sqrt(w)          normalized  v_s = sqrt(w / dw[s]), v_t = sqrt(w / dw[t])
// divided by sqrt(2) for a directed graph; float64 throughout, rounded once to T.
// Row i of D lists the edges incident to i in increasing edge id, which is the order the
// adjacency already gives: edges (j, i) with j < i come from rows j < i, then row i's own.
#include <cub/cub.cuh>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {

constexpr int kDiffThreads = 256;

static inline int diff_blocks(int64_t n) { return (int)ceil_div(n > 0 ? n : 1, kDiffThreads); }

// first position in [lo, hi) whose column is >= key
__device__ __forceinline__ int lower_bound_col(const int32_t* __restrict__ indices, int lo, int hi,
                                               int key) {
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(indices + mid) < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// value of D at (vertex, edge): sign -1 at the source, +1 at the target (difference.py:151-161)
template <typename T>
__device__ __forceinline__ T incidence_value(T w, double dw_vertex, int lap_type, bool directed,
                                             double sign) {
  double v = lap_type == 0 ? sqrt(double(w)) : sqrt(double(w) / dw_vertex);
  v = sign * v;
  if (directed) v = v / sqrt(2.0);
  return T(v);
}

// ---- edge offsets of an undirected graph: entries with col >= row, per row ----------------
__global__ void edge_offsets_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                    const int32_t* __restrict__ indices, int32_t* eptr) {
  const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row == 0) eptr[0] = 0;
  if (row >= n) return;
  const int end = __ldg(indptr + row + 1);
  eptr[row + 1] = end - lower_bound_col(indices, __ldg(indptr + row), end, (int)row);
}

// ---- edge list, and the row sizes of D^T (2, or 0 for a loop) into dt_indptr[k + 1] -------
// The edges of row i are the last eptr[i+1] - eptr[i] entries of the row.
template <typename T>
__global__ void edge_list_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                 const int32_t* __restrict__ indices, const T* __restrict__ data,
                                 const int32_t* __restrict__ eptr, int32_t* sources,
                                 int32_t* targets, T* weights, int32_t* dt_indptr) {
  const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row == 0) dt_indptr[0] = 0;
  if (row >= n) return;
  const int e0 = __ldg(eptr + row), e1 = __ldg(eptr + row + 1);
  const int k0 = __ldg(indptr + row + 1) - (e1 - e0);
  for (int e = e0, k = k0; e < e1; ++e, ++k) {
    const int col = __ldg(indices + k);
    sources[e] = (int32_t)row;
    targets[e] = col;
    weights[e] = __ldg(data + k);
    dt_indptr[e + 1] = col == row ? 0 : 2;
  }
}

// ---- D^T rows: one thread per edge ----------------------------------------------------------
template <typename T>
__global__ void incidence_t_kernel(int64_t ne, const int32_t* __restrict__ sources,
                                   const int32_t* __restrict__ targets,
                                   const T* __restrict__ weights, const double* __restrict__ dw,
                                   int lap_type, int directed, const int32_t* __restrict__ dt_indptr,
                                   int32_t* dt_indices, T* dt_data) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const int s = __ldg(sources + e), t = __ldg(targets + e);
  if (s == t) return;
  const T w = __ldg(weights + e);
  const double dws = lap_type == 1 ? __ldg(dw + s) : 0.0;
  const double dwt = lap_type == 1 ? __ldg(dw + t) : 0.0;
  const T vs = incidence_value<T>(w, dws, lap_type, directed != 0, -1.0);
  const T vt = incidence_value<T>(w, dwt, lap_type, directed != 0, +1.0);
  const int o = __ldg(dt_indptr + e);
  const bool s_first = s < t;
  dt_indices[o] = s_first ? s : t;
  dt_data[o] = s_first ? vs : vt;
  dt_indices[o + 1] = s_first ? t : s;
  dt_data[o + 1] = s_first ? vt : vs;
}

// ---- D rows: sizes ---------------------------------------------------------------------------
// Undirected: every non-loop entry of row i is one incident edge.  Directed: the non-loop entries
// of row i of W (out-edges) and of row i of W^T (in-edges).
__device__ __forceinline__ int non_loop_entries(const int32_t* __restrict__ indptr,
                                                const int32_t* __restrict__ indices, int64_t row) {
  const int start = __ldg(indptr + row), end = __ldg(indptr + row + 1);
  const int p = lower_bound_col(indices, start, end, (int)row);
  return (end - start) - (p < end && __ldg(indices + p) == row ? 1 : 0);
}

__global__ void incidence_count_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                       const int32_t* __restrict__ indices,
                                       const int32_t* __restrict__ t_indptr,
                                       const int32_t* __restrict__ t_indices, int32_t* d_indptr) {
  const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row == 0) d_indptr[0] = 0;
  if (row >= n) return;
  int c = non_loop_entries(indptr, indices, row);
  if (t_indptr) c += non_loop_entries(t_indptr, t_indices, row);
  d_indptr[row + 1] = c;
}

// ---- D rows: entries -----------------------------------------------------------------------
// Edge id of the entry (j, i) of W, found in row j:
//   undirected: its rank among row j's entries with col >= j, offset by eptr[j];
//   directed  : its position in W (eptr = indptr).
// Both are lower_bound(i in row j) - indptr[j+1] + eptr[j+1].
template <typename T>
__global__ void incidence_fill_kernel(int64_t n, int lap_type, const int32_t* __restrict__ indptr,
                                      const int32_t* __restrict__ indices,
                                      const T* __restrict__ data, const int32_t* __restrict__ eptr,
                                      const int32_t* __restrict__ t_indptr,
                                      const int32_t* __restrict__ t_indices,
                                      const T* __restrict__ t_data, const double* __restrict__ dw,
                                      const int32_t* __restrict__ d_indptr, int32_t* d_indices,
                                      T* d_data) {
  const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row >= n) return;
  const int i = (int)row;
  const bool directed = t_indptr != nullptr;
  const double dwi = lap_type == 1 ? __ldg(dw + row) : 0.0;
  // in-edges (j, i) come from W^T's row i when directed, else from W's row i (symmetric)
  const int32_t* in_ptr = directed ? t_indptr : indptr;
  const int32_t* in_idx = directed ? t_indices : indices;
  const T* in_val = directed ? t_data : data;
  const int in0 = __ldg(in_ptr + row), in1 = __ldg(in_ptr + row + 1);
  const int out0 = __ldg(indptr + row), out1 = __ldg(indptr + row + 1);
  int o = __ldg(d_indptr + row);

  auto in_edge = [&](int k) {                  // edge (j, i), j != i: vertex i is the target
    const int j = __ldg(in_idx + k);
    const int p = lower_bound_col(indices, __ldg(indptr + j), __ldg(indptr + j + 1), i);
    d_indices[o] = p - __ldg(indptr + j + 1) + __ldg(eptr + j + 1);
    d_data[o] = incidence_value<T>(__ldg(in_val + k), dwi, lap_type, directed, +1.0);
    ++o;
  };
  // in-edges from j < i: their ids lie in rows before i
  const int in_mid = lower_bound_col(in_idx, in0, in1, i);
  for (int k = in0; k < in_mid; ++k) in_edge(k);
  // out-edges (i, j): all of row i (directed) or its columns j > i (undirected), ids eptr[i]...
  const int first_out = directed ? out0 : lower_bound_col(indices, out0, out1, i);
  int e = __ldg(eptr + row);
  for (int k = first_out; k < out1; ++k, ++e) {
    const int j = __ldg(indices + k);
    if (j == i) continue;
    d_indices[o] = e;
    d_data[o] = incidence_value<T>(__ldg(data + k), dwi, lap_type, directed, -1.0);
    ++o;
  }
  // in-edges from j > i (directed only; undirected ones are the out-edges above)
  if (directed)
    for (int k = in_mid; k < in1; ++k)
      if (__ldg(in_idx + k) != i) in_edge(k);
}

// ------------------------------------------------------------------ drivers ------
int edge_offsets(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* eptr,
                 cudaStream_t st) {
  edge_offsets_kernel<<<diff_blocks(n), kDiffThreads, 0, st>>>(n, indptr, indices, eptr);
  GSP_LAUNCH_CHECK("edge_offsets");
  return scan_rows(eptr, n, st);
}

template <typename T>
int edge_list(int64_t n, int64_t ne, const int32_t* indptr, const int32_t* indices, const T* data,
              const int32_t* eptr, int32_t* sources, int32_t* targets, T* weights,
              int32_t* dt_indptr, cudaStream_t st) {
  edge_list_kernel<T><<<diff_blocks(n), kDiffThreads, 0, st>>>(n, indptr, indices, data, eptr,
                                                               sources, targets, weights,
                                                               dt_indptr);
  GSP_LAUNCH_CHECK("edge_list");
  return scan_rows(dt_indptr, ne, st);
}

template <typename T>
int incidence_t_fill(int64_t ne, const int32_t* sources, const int32_t* targets, const T* weights,
                     const double* dw, int lap_type, int directed, const int32_t* dt_indptr,
                     int32_t* dt_indices, T* dt_data, cudaStream_t st) {
  GSP_REQUIRE(lap_type == 0 || lap_type == 1, "Unknown Laplacian type");
  if (ne == 0) return GSP_OK;
  incidence_t_kernel<T><<<diff_blocks(ne), kDiffThreads, 0, st>>>(
      ne, sources, targets, weights, dw, lap_type, directed, dt_indptr, dt_indices, dt_data);
  GSP_LAUNCH_CHECK("incidence_t_fill");
  return GSP_OK;
}

int incidence_count(int64_t n, const int32_t* indptr, const int32_t* indices,
                    const int32_t* t_indptr, const int32_t* t_indices, int32_t* d_indptr,
                    cudaStream_t st) {
  incidence_count_kernel<<<diff_blocks(n), kDiffThreads, 0, st>>>(n, indptr, indices, t_indptr,
                                                                  t_indices, d_indptr);
  GSP_LAUNCH_CHECK("incidence_count");
  return scan_rows(d_indptr, n, st);
}

template <typename T>
int incidence_fill(int64_t n, int lap_type, const int32_t* indptr, const int32_t* indices,
                   const T* data, const int32_t* eptr, const int32_t* t_indptr,
                   const int32_t* t_indices, const T* t_data, const double* dw,
                   const int32_t* d_indptr, int32_t* d_indices, T* d_data, cudaStream_t st) {
  GSP_REQUIRE(lap_type == 0 || lap_type == 1, "Unknown Laplacian type");
  if (n == 0) return GSP_OK;
  incidence_fill_kernel<T><<<diff_blocks(n), kDiffThreads, 0, st>>>(
      n, lap_type, indptr, indices, data, eptr, t_indptr, t_indices, t_data, dw, d_indptr,
      d_indices, d_data);
  GSP_LAUNCH_CHECK("incidence_fill");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
#define GSP_DIFF_API(SUF, T)                                                                    \
  int gsp_edge_list_##SUF(int64_t n, int64_t n_edges, const int32_t* indptr,                    \
                          const int32_t* indices, const T* data, const int32_t* eptr,           \
                          int32_t* sources, int32_t* targets, T* weights, int32_t* dt_indptr,   \
                          void* stream) {                                                       \
    GSP_REQUIRE(n >= 0 && n_edges >= 0 && n_edges < (int64_t(1) << 31), "n_edges out of range"); \
    return gsp::edge_list<T>(n, n_edges, indptr, indices, data, eptr, sources, targets,         \
                             weights, dt_indptr, gsp::as_stream(stream));                       \
  }                                                                                             \
  int gsp_incidence_t_fill_##SUF(int64_t n_edges, const int32_t* sources,                       \
                                 const int32_t* targets, const T* weights, const double* dw,    \
                                 int lap_type, int directed, const int32_t* dt_indptr,          \
                                 int32_t* dt_indices, T* dt_data, void* stream) {               \
    return gsp::incidence_t_fill<T>(n_edges, sources, targets, weights, dw, lap_type, directed, \
                                    dt_indptr, dt_indices, dt_data, gsp::as_stream(stream));    \
  }                                                                                             \
  int gsp_incidence_fill_##SUF(int64_t n, int lap_type, const int32_t* indptr,                  \
                               const int32_t* indices, const T* data, const int32_t* eptr,      \
                               const int32_t* t_indptr, const int32_t* t_indices,               \
                               const T* t_data, const double* dw, const int32_t* d_indptr,      \
                               int32_t* d_indices, T* d_data, void* stream) {                   \
    return gsp::incidence_fill<T>(n, lap_type, indptr, indices, data, eptr, t_indptr,           \
                                  t_indices, t_data, dw, d_indptr, d_indices, d_data,           \
                                  gsp::as_stream(stream));                                      \
  }

extern "C" {
int gsp_edge_offsets(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* eptr,
                     void* stream) {
  GSP_REQUIRE(n >= 0, "n out of range");
  return gsp::edge_offsets(n, indptr, indices, eptr, gsp::as_stream(stream));
}
int gsp_incidence_count(int64_t n, const int32_t* indptr, const int32_t* indices,
                        const int32_t* t_indptr, const int32_t* t_indices, int32_t* d_indptr,
                        void* stream) {
  GSP_REQUIRE(n >= 0 && (t_indptr == nullptr) == (t_indices == nullptr), "bad arguments");
  return gsp::incidence_count(n, indptr, indices, t_indptr, t_indices, d_indptr,
                              gsp::as_stream(stream));
}
GSP_DIFF_API(f32, float)
GSP_DIFF_API(f64, double)
}
