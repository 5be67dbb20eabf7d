// Tree multiresolution (pygsp/reduction.py: tree_multiresolution, _tree_depths) on the device.
//
// Rooting: the 2 (n - 1) off-diagonal entries of a tree's symmetric adjacency are its arcs, in CSR
// order (gsp_tree_arc_count: per-row counts and their scan).  For the arc a = (u -> v), twin(a) is
// (v -> u), found by binary search in row v, and succ(a) is the arc after twin(a) in row v, wrapping
// round: the successors form one Euler circuit of the tree.  It is cut before the root's first arc,
// so the tour starts there, and ranked by Wyllie pointer jumping: ceil(log2 n_arcs) rounds of ping-pong
// (next, rank) pairs, a fixed count, so no host synchronisation.  pos(a) = n_arcs - 1 - rank(a) is
// a's place in the tour; a is downward iff pos(a) < pos(twin(a)).  A downward arc u -> v gives
// parent[v] = u and the weight to the parent w[v]; the depth is the inclusive scan of +1 (downward)
// and -1 (upward) over the tour, read at the downward arc into v.  O(log n) launches whatever the
// tree's depth (a path of n vertices has depth n - 1).
//
// Coarsening: keep the vertices of even depth (gsp_tree_keep: flags and their scan, the new ids);
// every kept non-root v, with p = parent[v] and g = parent[p], gets the edge (new(v), new(g)) whose
// weight combines w[v] and w[p] in double, rounded once to the graph's type (gsp_tree_coarsen_*),
// which also writes the next level's depth, parent and weight-to-parent arrays.  Only integer
// arithmetic and one double expression per edge: results are exact and reproducible.
#include <cub/cub.cuh>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {
namespace {

constexpr int kThreads = 256;
constexpr int32_t kEnd = -1;

inline int grid_of(int64_t n) { return (int)ceil_div(std::max<int64_t>(n, 1), kThreads); }

// first index i in [lo, hi) with a[i] >= key (hi when there is none)
__device__ __forceinline__ int64_t lower_bound(const int32_t* a, int64_t lo, int64_t hi,
                                               int32_t key) {
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// arc_ptr[0] = 0, arc_ptr[row + 1] = off-diagonal entries of the row (columns sorted, unique)
__global__ void arc_count_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                 const int32_t* __restrict__ indices, int32_t* arc_ptr) {
  const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (row == 0) arc_ptr[0] = 0;
  if (row >= n) return;
  const int64_t b = indptr[row], e = indptr[row + 1];
  const int64_t d = lower_bound(indices, b, e, (int32_t)row);
  arc_ptr[row + 1] = (int32_t)(e - b - (d < e && indices[d] == row ? 1 : 0));
}

// one thread per stored entry: its row by binary search over indptr, then its arc (diagonal skipped)
template <typename T>
__global__ void arc_fill_kernel(int64_t n, int64_t nnz, const int32_t* __restrict__ indptr,
                                const int32_t* __restrict__ indices, const T* __restrict__ data,
                                const int32_t* __restrict__ arc_ptr, int32_t* src, int32_t* dst,
                                double* wt) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= nnz) return;
  int64_t lo = 0, hi = n;                        // last row with indptr[row] <= e
  while (hi - lo > 1) {
    const int64_t mid = (lo + hi) >> 1;
    if (indptr[mid] <= e) lo = mid; else hi = mid;
  }
  const int64_t row = lo;
  const int32_t col = indices[e];
  if (col == row) return;
  const int64_t b = indptr[row];
  const bool has_diag = (indptr[row + 1] - b) != int64_t(arc_ptr[row + 1] - arc_ptr[row]);
  const int64_t a = arc_ptr[row] + (e - b) - (has_diag && col > row ? 1 : 0);
  src[a] = (int32_t)row;
  dst[a] = col;
  wt[a] = double(data[e]);
}

// twin and successor of every arc; the arc that would close the circuit ends the list
__global__ void tour_kernel(int64_t n_arcs, const int32_t* __restrict__ arc_ptr,
                            const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                            int32_t root, int32_t* twin, int2* link) {
  const int64_t a = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (a >= n_arcs) return;
  const int32_t u = src[a], v = dst[a];
  const int64_t b = arc_ptr[v], e = arc_ptr[v + 1];
  int64_t t = lower_bound(dst, b, e, u);
  if (t >= e || dst[t] != u) t = a;              // not a symmetric structure: no wild index
  twin[a] = (int32_t)t;
  const int64_t s = t + 1 < e ? t + 1 : b;
  link[a] = s == arc_ptr[root] ? make_int2(kEnd, 0) : make_int2((int32_t)s, 1);
}

// one Wyllie round: rank += rank of next, next = next of next
__global__ void wyllie_kernel(int64_t n_arcs, const int2* __restrict__ in, int2* out) {
  const int64_t a = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (a >= n_arcs) return;
  const int2 l = in[a];
  if (l.x == kEnd) {
    out[a] = l;
  } else {
    const int2 m = in[l.x];
    out[a] = make_int2(m.x, l.y + m.y);
  }
}

// step[pos(a)] = +1 / -1; a downward arc u -> v sets parent[v], w[v] and (for now) depth[v] = pos
__global__ void orient_kernel(int64_t n_arcs, const int32_t* __restrict__ src,
                              const int32_t* __restrict__ dst, const double* __restrict__ wt,
                              const int32_t* __restrict__ twin, const int2* __restrict__ link,
                              int32_t* step, int32_t* depth, int32_t* parent, double* wpar) {
  const int64_t a = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (a >= n_arcs) return;
  const int32_t pos = (int32_t)(n_arcs - 1 - link[a].y);
  const int32_t pos_twin = (int32_t)(n_arcs - 1 - link[twin[a]].y);
  const bool down = pos < pos_twin;
  step[pos] = down ? 1 : -1;
  if (down) {
    const int32_t v = dst[a];
    parent[v] = src[a];
    wpar[v] = wt[a];
    depth[v] = pos;
  }
}

__global__ void depth_kernel(int64_t n, int64_t n_arcs, int32_t root,
                             const int32_t* __restrict__ scan,
                             int32_t* depth, int32_t* parent, double* wpar) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= n) return;
  if (v == root) {
    depth[v] = 0;
    parent[v] = root;
    wpar[v] = 0.0;
  } else {
    const int32_t pos = depth[v];                // -1 unless a downward arc reached v
    depth[v] = pos >= 0 && pos < n_arcs ? scan[pos] : -1;
  }
}

// new_id[0] = 0, new_id[v + 1] = 1 when v's depth is even
__global__ void keep_flags_kernel(int64_t n, const int32_t* __restrict__ depth, int32_t* new_id) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v == 0) new_id[0] = 0;
  if (v >= n) return;
  new_id[v + 1] = (depth[v] & 1) == 0 ? 1 : 0;
}

__device__ __forceinline__ double combine(int method, double wv, double wp) {
  if (method == GSPB200_TREE_SUM) return __dadd_rn(wv, wp);
  if (method == GSPB200_TREE_RESISTANCE)
    return __ddiv_rn(1.0, __dadd_rn(__ddiv_rn(1.0, wv), __ddiv_rn(1.0, wp)));
  return 1.0;
}

template <typename T>
__global__ void coarsen_kernel(int64_t n, int64_t n_new, const int32_t* __restrict__ depth,
                               const int32_t* __restrict__ parent,
                               const double* __restrict__ wpar, const int32_t* __restrict__ new_id,
                               int32_t root, int method, int64_t* keep, int32_t* rows,
                               int32_t* cols, T* vals, int32_t* new_depth, int32_t* new_parent,
                               double* new_wpar) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int32_t d = depth[v];
  if (d & 1) return;
  const int32_t i = new_id[v];
  keep[i] = v;
  new_depth[i] = d >> 1;
  if (v == root) {
    new_parent[i] = i;
    new_wpar[i] = 0.0;
    return;
  }
  const int32_t p = parent[v], j = new_id[parent[p]];
  const T c = (T)combine(method, wpar[v], wpar[p]);
  new_parent[i] = j;
  new_wpar[i] = double(c);
  const int64_t m = n_new - 1;
  const int64_t e = i - (i > new_id[root] ? 1 : 0);
  rows[e] = i;
  cols[e] = j;
  vals[e] = c;
  rows[m + e] = j;
  cols[m + e] = i;
  vals[m + e] = c;
}

}  // namespace

int tree_arc_count(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* arc_ptr,
                   int64_t* n_arcs, cudaStream_t st) {
  arc_count_kernel<<<grid_of(n), kThreads, 0, st>>>(n, indptr, indices, arc_ptr);
  GSP_LAUNCH_CHECK("tree_arc_count");
  return scan_rows(arc_ptr, n, n_arcs, st);
}

template <typename T>
int tree_root(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
              const T* data, const int32_t* arc_ptr, int32_t root, int32_t* depth,
              int32_t* parent, double* wpar, cudaStream_t st) {
  const int64_t n_arcs = 2 * (n - 1);
  if (n_arcs > 0) {
    Scratch<int32_t> src(st), dst(st), twin(st), step(st);
    Scratch<double> wt(st);
    Scratch<int2> link(st), spare(st);
    GSP_CUDA(src.alloc(n_arcs));
    GSP_CUDA(dst.alloc(n_arcs));
    GSP_CUDA(twin.alloc(n_arcs));
    GSP_CUDA(step.alloc(n_arcs));
    GSP_CUDA(wt.alloc(n_arcs));
    GSP_CUDA(link.alloc(n_arcs));
    GSP_CUDA(spare.alloc(n_arcs));
    GSP_CUDA(cudaMemsetAsync(depth, 0xff, n * sizeof(int32_t), st));
    arc_fill_kernel<T><<<grid_of(nnz), kThreads, 0, st>>>(n, nnz, indptr, indices, data, arc_ptr,
                                                           src.get(), dst.get(), wt.get());
    GSP_LAUNCH_CHECK("tree_arc_fill");
    tour_kernel<<<grid_of(n_arcs), kThreads, 0, st>>>(n_arcs, arc_ptr, src.get(), dst.get(), root,
                                                      twin.get(), link.get());
    GSP_LAUNCH_CHECK("tree_tour");
    int2* cur = link.get();
    int2* nxt = spare.get();
    for (int64_t reach = 1; reach < n_arcs; reach *= 2) {
      wyllie_kernel<<<grid_of(n_arcs), kThreads, 0, st>>>(n_arcs, cur, nxt);
      GSP_LAUNCH_CHECK("tree_wyllie");
      std::swap(cur, nxt);
    }
    orient_kernel<<<grid_of(n_arcs), kThreads, 0, st>>>(n_arcs, src.get(), dst.get(), wt.get(),
                                                        twin.get(), cur, step.get(), depth, parent,
                                                        wpar);
    GSP_LAUNCH_CHECK("tree_orient");
    int32_t* s = step.get();
    const int rc = cub_temp("cub::DeviceScan::InclusiveSum", st, [&](void* tmp, size_t& bytes) {
      return cub::DeviceScan::InclusiveSum(tmp, bytes, s, s, (int)n_arcs, st);
    });
    if (rc != GSP_OK) return rc;
    depth_kernel<<<grid_of(n), kThreads, 0, st>>>(n, n_arcs, root, s, depth, parent, wpar);
    GSP_LAUNCH_CHECK("tree_depth");
    return GSP_OK;
  }
  depth_kernel<<<1, kThreads, 0, st>>>(n, 0, root, nullptr, depth, parent, wpar);
  GSP_LAUNCH_CHECK("tree_depth");
  return GSP_OK;
}

int tree_keep(int64_t n, const int32_t* depth, int32_t* new_id, int64_t* n_new, cudaStream_t st) {
  keep_flags_kernel<<<grid_of(n), kThreads, 0, st>>>(n, depth, new_id);
  GSP_LAUNCH_CHECK("tree_keep_flags");
  return scan_rows(new_id, n, n_new, st);
}

template <typename T>
int tree_coarsen(int64_t n, int64_t n_new, const int32_t* depth, const int32_t* parent,
                 const double* wpar, const int32_t* new_id, int32_t root, int method,
                 int64_t* keep, int32_t* rows, int32_t* cols, T* vals, int32_t* new_depth,
                 int32_t* new_parent, double* new_wpar, cudaStream_t st) {
  coarsen_kernel<T><<<grid_of(n), kThreads, 0, st>>>(n, n_new, depth, parent, wpar, new_id, root,
                                                     method, keep, rows, cols, vals, new_depth,
                                                     new_parent, new_wpar);
  GSP_LAUNCH_CHECK("tree_coarsen");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
#define GSP_TREE_OK_N(n) ((n) >= 1 && (n) <= (int64_t(1) << 30))

#define GSP_TREE_API(SUF, T)                                                                     \
  int gsp_tree_root_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,  \
                          const T* data, const int32_t* arc_ptr, int32_t root, int32_t* depth,   \
                          int32_t* parent, double* wpar, void* stream) {                         \
    GSP_REQUIRE(GSP_TREE_OK_N(n) && nnz >= 2 * (n - 1) && nnz < (int64_t(1) << 31) && root >= 0 \
                    && root < n && depth && parent && wpar,                                     \
                "bad arguments");                                                                \
    GSP_REQUIRE(n == 1 || (indptr && indices && data && arc_ptr), "no input");                   \
    return gsp::tree_root<T>(n, nnz, indptr, indices, data, arc_ptr, root, depth, parent, wpar,  \
                             gsp::as_stream(stream));                                            \
  }                                                                                              \
  int gsp_tree_coarsen_##SUF(int64_t n, int64_t n_new, const int32_t* depth,                      \
                             const int32_t* parent, const double* wpar, const int32_t* new_id,   \
                             int32_t root, int method, int64_t* keep, int32_t* rows,             \
                             int32_t* cols, T* vals, int32_t* new_depth, int32_t* new_parent,    \
                             double* new_wpar, void* stream) {                                   \
    GSP_REQUIRE(GSP_TREE_OK_N(n) && n_new >= 1 && n_new <= n && root >= 0 && root < n,          \
                "bad arguments");                                                                \
    GSP_REQUIRE(method == GSPB200_TREE_UNWEIGHTED || method == GSPB200_TREE_SUM ||               \
                    method == GSPB200_TREE_RESISTANCE,                                           \
                "unknown method");                                                               \
    GSP_REQUIRE(depth && parent && wpar && new_id && keep && new_depth && new_parent &&          \
                    new_wpar && (n_new == 1 || (rows && cols && vals)),                          \
                "no buffer");                                                                    \
    return gsp::tree_coarsen<T>(n, n_new, depth, parent, wpar, new_id, root, method, keep, rows, \
                                cols, vals, new_depth, new_parent, new_wpar,                     \
                                gsp::as_stream(stream));                                         \
  }

extern "C" {
int gsp_tree_arc_count(int64_t n, const int32_t* indptr, const int32_t* indices, int32_t* arc_ptr,
                       int64_t* n_arcs, void* stream) {
  GSP_REQUIRE(GSP_TREE_OK_N(n) && indptr && arc_ptr && n_arcs, "bad arguments");
  return gsp::tree_arc_count(n, indptr, indices, arc_ptr, n_arcs, gsp::as_stream(stream));
}
int gsp_tree_keep(int64_t n, const int32_t* depth, int32_t* new_id, int64_t* n_new,
                  void* stream) {
  GSP_REQUIRE(GSP_TREE_OK_N(n) && depth && new_id && n_new, "bad arguments");
  return gsp::tree_keep(n, depth, new_id, n_new, gsp::as_stream(stream));
}
GSP_TREE_API(f32, float)
GSP_TREE_API(f64, double)
}
