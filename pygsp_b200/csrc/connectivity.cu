// Graph connectivity: component labels, reachability from one vertex, induced subgraphs and
// the split of a graph into its components, all in HBM from a canonical CSR adjacency.
//
// Replaces, for pygsp/graphs/graph.py:
//   * the Python BFS of is_connected (:340-366) and extract_components (:478-500), one vertex
//     and one `W[v].nonzero()` at a time;
//   * W[vertices, :][:, vertices] of subgraph (:247), SciPy fancy indexing.
//
// Component labels are union-find over the entries with col > row, in the style of ECL-CC
// (Jaiganesh and Burtscher, HPDC 2018): a thread per row hooks the larger of two roots under
// the smaller with atomicCAS, `find` halves the path it walks, a last pass writes every
// vertex's root.  Parents only ever point to smaller ids, so the root of a tree is the smallest
// vertex of its component whatever the scheduling: the labels are deterministic, and the work
// does not depend on the diameter (label propagation does).
//
// Reachability (directed is_connected) is a level-synchronous frontier BFS.  A launch runs one
// level; the entry point enqueues a bounded batch of levels and the caller reads one small
// state block per batch, so there is no host round trip per level.  Its cost is proportional
// to the diameter, which is inherent to the level-synchronous form.
//
// Subgraphs are count -> scan -> fill through a multiplicity map of the kept vertices (for each
// old vertex, the new positions that hold it, in increasing order).
#include <cub/cub.cuh>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {

constexpr int kConnThreads = 256;

static inline int conn_blocks(int64_t n) { return (int)ceil_div(n > 0 ? n : 1, kConnThreads); }

// number of bits that hold every value in [0, n)
static inline int key_bits(int64_t n) {
  int bits = 1;
  while ((int64_t(1) << bits) < n && bits < 31) ++bits;
  return bits;
}

// ---- union-find ------------------------------------------------------------------------------
// Invariant: parent[x] <= x, and parent[x] == x only at a root.  Halving writes go to non-roots
// only and store an ancestor, so they never undo a hook; a hook (atomicCAS) succeeds on a root
// only.  Reads go through a volatile pointer: other threads rewrite parents during the launch.
// The last pass must not halve: a late halving store could replace a vertex's final label (its
// root) with an ancestor read before that label was written.
template <bool HALVE>
__device__ __forceinline__ int find_root(int32_t* parent, int x) {
  volatile int32_t* p = parent;
  int cur = p[x];
  if (cur == x) return x;
  int prev = x, next;
  while (cur > (next = p[cur])) {
    if (HALVE) p[prev] = next;
    prev = cur;
    cur = next;
  }
  return cur;
}

__device__ __forceinline__ void unite(int32_t* parent, int a, int b) {
  int ra = find_root<true>(parent, a), rb = find_root<true>(parent, b);
  while (ra != rb) {
    const int hi = ra > rb ? ra : rb, lo = ra > rb ? rb : ra;
    const int old = atomicCAS(parent + hi, hi, lo);
    if (old == hi) return;
    // hi was hooked by another thread meanwhile: continue from its new root
    if (ra == hi) ra = find_root<true>(parent, old); else rb = find_root<true>(parent, old);
  }
}

__global__ void cc_init_kernel(int64_t n, int32_t* parent) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v < n) parent[v] = (int32_t)v;
}

template <typename T>
__global__ void cc_hook_kernel(int64_t n, const int32_t* __restrict__ indptr,
                               const int32_t* __restrict__ indices, const T* __restrict__ data,
                               int positive_only, int32_t* parent) {
  const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row >= n) return;
  const int end = __ldg(indptr + row + 1);
  for (int k = __ldg(indptr + row); k < end; ++k) {
    const int col = __ldg(indices + k);
    if (col <= row) continue;
    if (positive_only && !(__ldg(data + k) > T(0))) continue;
    unite(parent, (int)row, col);
  }
}

__global__ void cc_finish_kernel(int64_t n, int32_t* parent, unsigned long long* n_components) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  bool root = false;
  if (v < n) {
    const int r = find_root<false>(parent, (int)v);
    parent[v] = r;
    root = r == (int)v;
  }
  const unsigned roots = __popc(__ballot_sync(0xffffffffu, root));
  if (n_components && (threadIdx.x & 31) == 0 && roots) atomicAdd(n_components, roots);
}

// ---- reachability: one BFS level per launch ---------------------------------------------------
// state[0..2]: frontier sizes of levels L, L+1, L+2 (a ring indexed by level % 3), state[3]:
// vertices of the levels done so far.  Level L reads its frontier from queue half L & 1 and
// appends the next one to the other half; it also clears the slot level L + 2 will append to.
__global__ void reach_init_kernel(int32_t source, int32_t* visited, int32_t* queue,
                                  unsigned long long* state) {
  visited[source] = 1;
  queue[0] = source;
  state[0] = 1;
}

__global__ void reach_level_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                   const int32_t* __restrict__ indices, int32_t* visited,
                                   int32_t* queue, unsigned long long* state, int64_t level) {
  const int64_t size = (int64_t)state[level % 3];
  unsigned long long* next_size = state + (level + 1) % 3;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    state[(level + 2) % 3] = 0;
    state[3] += (unsigned long long)size;
  }
  const int32_t* cur = queue + (level & 1) * n;
  int32_t* nxt = queue + ((level + 1) & 1) * n;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < size; i += stride) {
    const int v = cur[i];
    const int end = __ldg(indptr + v + 1);
    for (int k = __ldg(indptr + v); k < end; ++k) {
      const int u = __ldg(indices + k);
      if (visited[u] == 0 && atomicExch(visited + u, 1) == 0)
        nxt[atomicAdd(next_size, 1ull)] = u;
    }
  }
}

// ---- multiplicity map and induced subgraph ----------------------------------------------------
__global__ void vertex_count_kernel(int64_t m, const int32_t* __restrict__ v, int32_t* mptr) {
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (p < m) atomicAdd(mptr + __ldg(v + p) + 1, 1);
}

__global__ void iota_kernel(int64_t n, int32_t* out) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (int32_t)i;
}

// kept entries of new row r (old row v[r]): the multiplicities of its columns, restricted to the
// columns with the row's label when labels are given
__global__ void subgraph_count_kernel(int64_t m, const int32_t* __restrict__ indptr,
                                      const int32_t* __restrict__ indices,
                                      const int32_t* __restrict__ v,
                                      const int32_t* __restrict__ mptr,
                                      const int32_t* __restrict__ labels, int32_t* s_indptr) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r == 0) s_indptr[0] = 0;
  if (r >= m) return;
  const int u = __ldg(v + r);
  const int lu = labels ? __ldg(labels + u) : 0;
  const int end = __ldg(indptr + u + 1);
  int s = 0;                               // at most m < 2^31: the columns of a row are distinct
  for (int k = __ldg(indptr + u); k < end; ++k) {
    const int c = __ldg(indices + k);
    if (labels && __ldg(labels + c) != lu) continue;
    s += __ldg(mptr + c + 1) - __ldg(mptr + c);
  }
  s_indptr[r + 1] = s;
}

template <typename T>
__global__ void subgraph_fill_kernel(int64_t m, const int32_t* __restrict__ indptr,
                                     const int32_t* __restrict__ indices,
                                     const T* __restrict__ data, const int32_t* __restrict__ v,
                                     const int32_t* __restrict__ mptr,
                                     const int32_t* __restrict__ mpos,
                                     const int32_t* __restrict__ labels,
                                     const int32_t* __restrict__ s_indptr, int32_t* s_indices,
                                     T* s_data, int32_t* s_rows) {
  const int64_t r = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (r >= m) return;
  const int u = __ldg(v + r);
  const int lu = labels ? __ldg(labels + u) : 0;
  const int end = __ldg(indptr + u + 1);
  int o = __ldg(s_indptr + r);
  for (int k = __ldg(indptr + u); k < end; ++k) {
    const int c = __ldg(indices + k);
    if (labels && __ldg(labels + c) != lu) continue;
    const T w = __ldg(data + k);
    const int q1 = __ldg(mptr + c + 1);
    for (int q = __ldg(mptr + c); q < q1; ++q, ++o) {
      s_indices[o] = __ldg(mpos + q);
      s_data[o] = w;
      if (s_rows) s_rows[o] = (int32_t)r;
    }
  }
}

// ---- components in order: first position of each component in the sorted vertex order -------
__global__ void root_flags_kernel(int64_t n, const int32_t* __restrict__ labels, int32_t* rank) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v == 0) rank[0] = 0;
  if (v < n) rank[v + 1] = __ldg(labels + v) == v ? 1 : 0;
}

__global__ void component_starts_kernel(int64_t n, const int32_t* __restrict__ sorted_labels,
                                        const int32_t* __restrict__ rank, int32_t* comp_ptr,
                                        int64_t* n_components) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int key = __ldg(sorted_labels + i);
  if (i == 0 || __ldg(sorted_labels + i - 1) != key) comp_ptr[__ldg(rank + key)] = (int32_t)i;
  if (i == 0) {
    const int nc = __ldg(rank + n);
    comp_ptr[nc] = (int32_t)n;
    if (n_components) *n_components = nc;
  }
}

// ---- is_weighted -------------------------------------------------------------------------------
template <typename T>
__global__ void not_one_kernel(int64_t nnz, const T* __restrict__ data, int32_t* flag) {
  bool any = false;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < nnz;
       i += int64_t(gridDim.x) * blockDim.x)
    any |= __ldg(data + i) != T(1);
  if (__any_sync(0xffffffffu, any) && (threadIdx.x & 31) == 0) *flag = 1;
}

// ------------------------------------------------------------------ drivers ------
template <typename T>
int cc_labels(int64_t n, const int32_t* indptr, const int32_t* indices, const T* data,
              int positive_only, int32_t* labels, int64_t* n_components, cudaStream_t st) {
  if (n_components) GSP_CUDA(cudaMemsetAsync(n_components, 0, sizeof(int64_t), st));
  if (n == 0) return GSP_OK;
  cc_init_kernel<<<conn_blocks(n), kConnThreads, 0, st>>>(n, labels);
  GSP_LAUNCH_CHECK("cc_init");
  cc_hook_kernel<T><<<conn_blocks(n), kConnThreads, 0, st>>>(n, indptr, indices, data,
                                                            positive_only, labels);
  GSP_LAUNCH_CHECK("cc_hook");
  cc_finish_kernel<<<conn_blocks(n), kConnThreads, 0, st>>>(
      n, labels, reinterpret_cast<unsigned long long*>(n_components));
  GSP_LAUNCH_CHECK("cc_finish");
  return GSP_OK;
}

int reach_init(int64_t n, int32_t source, int32_t* visited, int32_t* queue, int64_t* state,
               cudaStream_t st) {
  GSP_CUDA(cudaMemsetAsync(visited, 0, sizeof(int32_t) * n, st));
  GSP_CUDA(cudaMemsetAsync(state, 0, sizeof(int64_t) * 4, st));
  reach_init_kernel<<<1, 1, 0, st>>>(source, visited, queue,
                                     reinterpret_cast<unsigned long long*>(state));
  GSP_LAUNCH_CHECK("reach_init");
  return GSP_OK;
}

int reach_levels(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* visited,
                 int32_t* queue, int64_t* state, int64_t level0, int n_levels, cudaStream_t st) {
  const int blocks = (int)std::min<int64_t>(conn_blocks(n), 4 * int64_t(sm_count()));
  for (int l = 0; l < n_levels; ++l) {
    reach_level_kernel<<<blocks, kConnThreads, 0, st>>>(
        n, indptr, indices, visited, queue, reinterpret_cast<unsigned long long*>(state),
        level0 + l);
    GSP_LAUNCH_CHECK("reach_level");
  }
  return GSP_OK;
}

int vertex_map(int64_t n, int64_t m, const int32_t* v, int32_t* mptr, int32_t* mpos,
               cudaStream_t st) {
  GSP_CUDA(cudaMemsetAsync(mptr, 0, sizeof(int32_t) * (n + 1), st));
  if (m == 0) return GSP_OK;
  vertex_count_kernel<<<conn_blocks(m), kConnThreads, 0, st>>>(m, v, mptr);
  GSP_LAUNCH_CHECK("vertex_count");
  int rc = scan_rows(mptr, n, nullptr, st);
  if (rc != GSP_OK) return rc;
  // positions sorted by old id; the radix sort is stable, so each old id's positions increase
  Scratch<int32_t> pos(st), keys_out(st);
  GSP_CUDA(pos.alloc(m));
  GSP_CUDA(keys_out.alloc(m));
  iota_kernel<<<conn_blocks(m), kConnThreads, 0, st>>>(m, pos.get());
  GSP_LAUNCH_CHECK("iota");
  return cub_temp("cub::DeviceRadixSort::SortPairs", st, [&](void* tmp, size_t& bytes) {
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, v, keys_out.get(), pos.get(), mpos, (int)m,
                                           0, key_bits(n), st);
  });
}

int subgraph_count(int64_t m, const int32_t* indptr, const int32_t* indices, const int32_t* v,
                   const int32_t* mptr, const int32_t* labels, int32_t* s_indptr, int64_t* nnz,
                   cudaStream_t st) {
  subgraph_count_kernel<<<conn_blocks(m), kConnThreads, 0, st>>>(m, indptr, indices, v, mptr,
                                                                  labels, s_indptr);
  GSP_LAUNCH_CHECK("subgraph_count");
  return scan_rows(s_indptr, m, nnz, st);
}

template <typename T>
int subgraph_fill(int64_t m, const int32_t* indptr, const int32_t* indices, const T* data,
                  const int32_t* v, const int32_t* mptr, const int32_t* mpos,
                  const int32_t* labels, const int32_t* s_indptr, int32_t* s_indices, T* s_data,
                  int32_t* s_rows, cudaStream_t st) {
  if (m == 0) return GSP_OK;
  subgraph_fill_kernel<T><<<conn_blocks(m), kConnThreads, 0, st>>>(
      m, indptr, indices, data, v, mptr, mpos, labels, s_indptr, s_indices, s_data, s_rows);
  GSP_LAUNCH_CHECK("subgraph_fill");
  return GSP_OK;
}

int component_order(int64_t n, const int32_t* labels, int32_t* perm, int32_t* comp_ptr,
                     int64_t* n_components, cudaStream_t st) {
  if (n == 0) {
    GSP_CUDA(cudaMemsetAsync(comp_ptr, 0, sizeof(int32_t), st));
    if (n_components) GSP_CUDA(cudaMemsetAsync(n_components, 0, sizeof(int64_t), st));
    return GSP_OK;
  }
  Scratch<int32_t> ids(st), sorted(st), rank(st);
  GSP_CUDA(ids.alloc(n));
  GSP_CUDA(sorted.alloc(n));
  GSP_CUDA(rank.alloc(n + 1));
  iota_kernel<<<conn_blocks(n), kConnThreads, 0, st>>>(n, ids.get());
  GSP_LAUNCH_CHECK("iota");
  root_flags_kernel<<<conn_blocks(n), kConnThreads, 0, st>>>(n, labels, rank.get());
  GSP_LAUNCH_CHECK("root_flags");
  // vertices by (label, id): a stable sort of the labels
  int rc = cub_temp("cub::DeviceRadixSort::SortPairs", st, [&](void* tmp, size_t& bytes) {
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, labels, sorted.get(), ids.get(), perm,
                                           (int)n, 0, key_bits(n), st);
  });
  if (rc != GSP_OK) return rc;
  rc = scan_rows(rank.get(), n, nullptr, st);
  if (rc != GSP_OK) return rc;
  component_starts_kernel<<<conn_blocks(n), kConnThreads, 0, st>>>(n, sorted.get(), rank.get(),
                                                                   comp_ptr, n_components);
  GSP_LAUNCH_CHECK("component_starts");
  return GSP_OK;
}

template <typename T>
int weights_not_one(int64_t nnz, const T* data, int32_t* flag, cudaStream_t st) {
  GSP_CUDA(cudaMemsetAsync(flag, 0, sizeof(int32_t), st));
  if (nnz == 0) return GSP_OK;
  const int blocks = (int)std::min<int64_t>(conn_blocks(nnz), 4 * int64_t(sm_count()));
  not_one_kernel<T><<<blocks, kConnThreads, 0, st>>>(nnz, data, flag);
  GSP_LAUNCH_CHECK("weights_not_one");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
#define GSP_CONN_API(SUF, T)                                                                    \
  int gsp_cc_labels_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,             \
                          const T* data, int positive_only, int32_t* labels,                    \
                          int64_t* n_components, void* stream) {                                \
    GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31), "n out of range");                          \
    return gsp::cc_labels<T>(n, indptr, indices, data, positive_only, labels, n_components,     \
                             gsp::as_stream(stream));                                           \
  }                                                                                             \
  int gsp_subgraph_fill_##SUF(int64_t m, const int32_t* indptr, const int32_t* indices,         \
                              const T* data, const int32_t* v, const int32_t* mptr,             \
                              const int32_t* mpos, const int32_t* labels,                       \
                              const int32_t* s_indptr, int32_t* s_indices, T* s_data,           \
                              int32_t* s_rows, void* stream) {                                  \
    GSP_REQUIRE(m >= 0 && m < (int64_t(1) << 31), "m out of range");                           \
    return gsp::subgraph_fill<T>(m, indptr, indices, data, v, mptr, mpos, labels, s_indptr,     \
                                 s_indices, s_data, s_rows, gsp::as_stream(stream));            \
  }                                                                                             \
  int gsp_weights_not_one_##SUF(int64_t nnz, const T* data, int32_t* flag, void* stream) {      \
    GSP_REQUIRE(nnz >= 0, "nnz out of range");                                                  \
    return gsp::weights_not_one<T>(nnz, data, flag, gsp::as_stream(stream));                    \
  }

extern "C" {
int gsp_reach_init(int64_t n, int32_t source, int32_t* visited, int32_t* queue, int64_t* state,
                   void* stream) {
  GSP_REQUIRE(n > 0 && n < (int64_t(1) << 31) && source >= 0 && source < n, "bad arguments");
  return gsp::reach_init(n, source, visited, queue, state, gsp::as_stream(stream));
}
int gsp_reach_levels(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* visited,
                     int32_t* queue, int64_t* state, int64_t level0, int n_levels, void* stream) {
  GSP_REQUIRE(n > 0 && n < (int64_t(1) << 31) && level0 >= 0 && n_levels >= 0, "bad arguments");
  return gsp::reach_levels(n, indptr, indices, visited, queue, state, level0, n_levels,
                           gsp::as_stream(stream));
}
int gsp_vertex_map(int64_t n, int64_t m, const int32_t* v, int32_t* mptr, int32_t* mpos,
                   void* stream) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31) && m >= 0 && m < (int64_t(1) << 31),
              "bad arguments");
  return gsp::vertex_map(n, m, v, mptr, mpos, gsp::as_stream(stream));
}
int gsp_subgraph_count(int64_t m, const int32_t* indptr, const int32_t* indices, const int32_t* v,
                       const int32_t* mptr, const int32_t* labels, int32_t* s_indptr,
                       int64_t* nnz, void* stream) {
  GSP_REQUIRE(m >= 0 && m < (int64_t(1) << 31), "m out of range");
  return gsp::subgraph_count(m, indptr, indices, v, mptr, labels, s_indptr, nnz,
                             gsp::as_stream(stream));
}
int gsp_component_order(int64_t n, const int32_t* labels, int32_t* perm, int32_t* comp_ptr,
                        int64_t* n_components, void* stream) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31), "n out of range");
  return gsp::component_order(n, labels, perm, comp_ptr, n_components, gsp::as_stream(stream));
}
GSP_CONN_API(f32, float)
GSP_CONN_API(f64, double)
}
