// Barnes-Hut repulsion of the Fruchterman-Reingold layout (DESIGN.md 4.24): the sum
// k^2 sum_j (p_i - p_j) / max(|p_i - p_j|^2, 0.01^2) of csrc/layout.cu in O(n log n), float64,
// dim 1, 2 or 3.  One iteration:
//
//   1. bh_box_partial_kernel / bh_box_final_kernel: per-axis min and max of the positions (a
//      min/max reduction: exact, independent of order); span = max(hi - lo, 1e-300).
//   2. bh_keys_kernel: Morton keys with the quantisation of graphs.morton_order: 21 bits per axis,
//      q = trunc((x - lo) / span * 2^21) in float64, clamped to [0, 2^21 - 1]; NaN gives 0.
//   3. cub::DeviceRadixSort::SortPairs of (key, id) over the 21 dim key bits: stable, so equal
//      keys stay in id order.  bh_gather_kernel copies the positions into sorted order (spos).
//   4. bh_build_kernel: Karras's binary radix tree (HPG 2012) over the sorted keys, a duplicate
//      key broken by its sorted index.  Internal node i (0 <= i < n - 1) covers the sorted range
//      [min(i, j), max(i, j)]; its split g is the last index of the left child.  A child is a
//      leaf when its range is one index: children store v >= 0 for internal node v and ~s (< 0)
//      for the leaf at sorted index s.  The root is internal node 0, or leaf ~0 when n = 1.  The
//      numbering is a function of the key ranges alone (a node covering [a, b] is numbered b
//      when it is its parent's left child, a when it is the right child).
//   5. bh_aggregate_kernel: one thread per leaf climbs to the root; the second child to arrive
//      at a node finishes it (count, AABB of the real points, centroid), left child then right
//      child, so the bits do not depend on timing.  Writes are published by __threadfence before
//      the flag's atomicAdd, and the sibling's data are read with ld.global.cg (L2, coherent).
//      The centroid is c = c_L + (M_R / M) (c_R - c_L): every cell's centroid is relative to a
//      member point, so a cell of coincident points has their exact position.
//   6. bh_walk_kernel<DIM>: one thread per query, in sorted order (a warp's walks coincide).  A
//      depth-first walk with an explicit stack, left child before right, fixes each vertex's
//      summation order.  A cell with count M, centroid c, AABB diagonal D and distance rho from
//      the query to its AABB is one monopole M f(x - c), f(r) = r / max(|r|^2, 0.01^2), when
//      D <= theta rho and rho >= 0.01, or when its AABB is one point (D = 0, exact); otherwise it
//      is opened.  A leaf adds f(x - y) exactly as the all-pairs kernel does (the self pair and
//      duplicates add exact zeros); k^2 multiplies once at the end.  partial[id] receives the
//      sum in the caller's vertex order.
//   7. spring_update_kernel<T> (csrc/spring.cuh) with one chunk.
//
// Bounds.  Every index the build computes is i + l d with delta(i, .) = -1 outside [0, n), so the
// searches stay in range; n < 2^31 so sorted indices fit the 31 id bits.  The extended key (21 dim
// Morton bits, then 31 index bits) is distinct per leaf, and the prefix lengths of the nodes on a
// root-to-leaf path strictly increase through the 21 dim + 31 <= 94 values delta can take for
// them, so the depth is at most 94 and the walk's stack (one pending right child per level)
// never holds more than 94 entries.  The guard below can therefore not fire; if it did it would
// set the status that the entry point returns as an error.
#include <cub/cub.cuh>
#include <math.h>

#include "common.cuh"
#include "gspb200.h"
#include "spring.cuh"

namespace gsp {
namespace {

using spring::inv_d2;
using spring::kMinD2;

constexpr int kAxisBits = 21;              // Morton bits per axis (graphs.morton_order, dim <= 3)
constexpr int kIdBits = 31;                // sorted indices: n < 2^31
constexpr int kStack = 96;                 // walk stack entries
static_assert(kStack >= kAxisBits * 3 + kIdBits,
              "the walk stack must hold one entry per level of the deepest tree");
constexpr int kBoxBlocks = 264;            // CTAs of the bounding-box reduction (a constant)
constexpr int kBoxThreads = 256;
constexpr int kWalkThreads = 128;
constexpr double kQuant = double(1 << kAxisBits);

// internal-node record: lo[DIM], hi[DIM], centroid[DIM], count (as double), children (int2)
template <int DIM>
__host__ __device__ constexpr int rec_len() { return 3 * DIM + 2; }

template <int DIM>
__global__ void __launch_bounds__(kBoxThreads)
    bh_box_partial_kernel(int64_t n, const double* __restrict__ pos, double* __restrict__ part) {
  __shared__ double s[2 * DIM][kBoxThreads];
  double lo[DIM], hi[DIM];
#pragma unroll
  for (int a = 0; a < DIM; ++a) {
    lo[a] = INFINITY;
    hi[a] = -INFINITY;
  }
  for (int64_t i = int64_t(blockIdx.x) * kBoxThreads + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * kBoxThreads) {
#pragma unroll
    for (int a = 0; a < DIM; ++a) {
      const double v = pos[i * DIM + a];
      lo[a] = fmin(lo[a], v);
      hi[a] = fmax(hi[a], v);
    }
  }
#pragma unroll
  for (int a = 0; a < DIM; ++a) {
    s[a][threadIdx.x] = lo[a];
    s[DIM + a][threadIdx.x] = hi[a];
  }
  for (int w = kBoxThreads / 2; w > 0; w /= 2) {
    __syncthreads();
    if (threadIdx.x < w) {
#pragma unroll
      for (int a = 0; a < DIM; ++a) {
        s[a][threadIdx.x] = fmin(s[a][threadIdx.x], s[a][threadIdx.x + w]);
        s[DIM + a][threadIdx.x] = fmax(s[DIM + a][threadIdx.x], s[DIM + a][threadIdx.x + w]);
      }
    }
  }
  __syncthreads();   // thread 0's last combine is visible to the writers below
  if (threadIdx.x < 2 * DIM) part[blockIdx.x * 2 * DIM + threadIdx.x] = s[threadIdx.x][0];
}

// box[0, DIM) = lo, box[DIM, 2 DIM) = span = max(hi - lo, 1e-300) (graphs.morton_order)
template <int DIM>
__global__ void bh_box_final_kernel(int parts, const double* __restrict__ part,
                                    double* __restrict__ box) {
  const int a = threadIdx.x;
  if (a >= DIM) return;
  double lo = INFINITY, hi = -INFINITY;
  for (int b = 0; b < parts; ++b) {
    lo = fmin(lo, part[b * 2 * DIM + a]);
    hi = fmax(hi, part[b * 2 * DIM + DIM + a]);
  }
  box[a] = lo;
  box[DIM + a] = fmax(hi - lo, 1e-300);
}

template <int DIM>
__global__ void bh_keys_kernel(int64_t n, const double* __restrict__ pos,
                               const double* __restrict__ box, uint64_t* __restrict__ keys,
                               int32_t* __restrict__ ids) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t code = 0;
#pragma unroll
  for (int a = 0; a < DIM; ++a) {
    const double v = (pos[i * DIM + a] - box[a]) / box[DIM + a] * kQuant;
    // truncation toward zero, clamped; a NaN fails `v > 0` and quantises to 0
    const uint64_t q = v > 0.0 ? (v < kQuant ? uint64_t(v) : uint64_t((1 << kAxisBits) - 1)) : 0;
#pragma unroll
    for (int b = 0; b < kAxisBits; ++b) code |= ((q >> b) & 1ull) << (b * DIM + a);
  }
  keys[i] = code;
  ids[i] = int32_t(i);
}

// spos[s] = pos[ids[s]]; the aggregation flags start at 0
template <int DIM>
__global__ void bh_gather_kernel(int64_t n, const double* __restrict__ pos,
                                 const int32_t* __restrict__ ids, double* __restrict__ spos,
                                 int32_t* __restrict__ flags) {
  const int64_t s = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int64_t id = ids[s];
#pragma unroll
  for (int a = 0; a < DIM; ++a) spos[s * DIM + a] = pos[id * DIM + a];
  if (s < n - 1) flags[s] = 0;
}

// common prefix length of the extended keys (key_i, i) and (key_j, j); -1 outside [0, n)
__device__ __forceinline__ int bh_delta(const uint64_t* __restrict__ keys, int64_t n, int64_t i,
                                        int64_t j) {
  if (j < 0 || j >= n) return -1;
  const uint64_t a = keys[i], b = keys[j];
  if (a != b) return __clzll((long long)(a ^ b));
  return 64 + __clz(int(uint32_t(i) ^ uint32_t(j)));
}

// Karras's construction for internal node i; parent[v] of internal node v, parent[n - 1 + s] of
// the leaf at sorted index s (-1 for the root)
template <int DIM>
__global__ void bh_build_kernel(int64_t n, const uint64_t* __restrict__ keys,
                                double* __restrict__ rec, int32_t* __restrict__ parent) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n - 1) return;
  const int d = bh_delta(keys, n, i, i + 1) - bh_delta(keys, n, i, i - 1) > 0 ? 1 : -1;
  const int dmin = bh_delta(keys, n, i, i - d);
  int64_t lmax = 2;
  while (bh_delta(keys, n, i, i + lmax * d) > dmin) lmax *= 2;
  int64_t l = 0;
  for (int64_t t = lmax / 2; t >= 1; t /= 2)
    if (bh_delta(keys, n, i, i + (l + t) * d) > dmin) l += t;
  const int64_t j = i + l * d;
  const int dnode = bh_delta(keys, n, i, j);
  int64_t s = 0, t = l;
  do {
    t = (t + 1) / 2;
    if (bh_delta(keys, n, i, i + (s + t) * d) > dnode) s += t;
  } while (t > 1);
  const int64_t g = i + s * d + min(d, 0);
  const int32_t left = min(i, j) == g ? ~int32_t(g) : int32_t(g);
  const int32_t right = max(i, j) == g + 1 ? ~int32_t(g + 1) : int32_t(g + 1);
  *reinterpret_cast<int2*>(rec + i * rec_len<DIM>() + 3 * DIM + 1) = make_int2(left, right);
  parent[left < 0 ? n - 1 + ~left : left] = int32_t(i);
  parent[right < 0 ? n - 1 + ~right : right] = int32_t(i);
  if (i == 0) parent[0] = -1;
}

template <int DIM>
struct Cell {
  double lo[DIM], hi[DIM], c[DIM];
  int64_t m;
};

template <int DIM>
__device__ __forceinline__ Cell<DIM> bh_load_cell(int32_t v, const double* spos,
                                                  const double* rec) {
  Cell<DIM> x;
  if (v < 0) {
#pragma unroll
    for (int a = 0; a < DIM; ++a) x.lo[a] = x.hi[a] = x.c[a] = spos[int64_t(~v) * DIM + a];
    x.m = 1;
  } else {
    const double* r = rec + int64_t(v) * rec_len<DIM>();
#pragma unroll
    for (int a = 0; a < DIM; ++a) {
      x.lo[a] = __ldcg(r + a);
      x.hi[a] = __ldcg(r + DIM + a);
      x.c[a] = __ldcg(r + 2 * DIM + a);
    }
    x.m = int64_t(__ldcg(r + 3 * DIM));
  }
  return x;
}

template <int DIM>
__global__ void bh_aggregate_kernel(int64_t n, const double* __restrict__ spos, double* rec,
                                    const int32_t* __restrict__ parent, int32_t* flags) {
  const int64_t s = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (s >= n) return;
  int32_t v = parent[n - 1 + s];
  while (v >= 0) {
    __threadfence();                             // this thread's node is visible before its flag
    if (atomicAdd(flags + v, 1) == 0) return;    // the sibling is not done: it finishes v
    __threadfence();
    double* r = rec + int64_t(v) * rec_len<DIM>();
    const int2 ch = *reinterpret_cast<const int2*>(r + 3 * DIM + 1);
    const Cell<DIM> L = bh_load_cell<DIM>(ch.x, spos, rec);
    const Cell<DIM> R = bh_load_cell<DIM>(ch.y, spos, rec);
    const int64_t m = L.m + R.m;
    const double w = double(R.m) / double(m);
#pragma unroll
    for (int a = 0; a < DIM; ++a) {
      r[a] = fmin(L.lo[a], R.lo[a]);
      r[DIM + a] = fmax(L.hi[a], R.hi[a]);
      r[2 * DIM + a] = fma(w, R.c[a] - L.c[a], L.c[a]);
    }
    r[3 * DIM] = double(m);
    v = parent[v];
  }
}

template <int DIM>
__global__ void __launch_bounds__(kWalkThreads)
    bh_walk_kernel(int64_t n, const double* __restrict__ spos, const int32_t* __restrict__ ids,
                   const double* __restrict__ rec, double theta2, double k2,
                   double* __restrict__ partial, int32_t* __restrict__ status) {
  const int64_t s = int64_t(blockIdx.x) * kWalkThreads + threadIdx.x;
  if (s >= n) return;
  double x[DIM], acc[DIM];
#pragma unroll
  for (int a = 0; a < DIM; ++a) {
    x[a] = spos[s * DIM + a];
    acc[a] = 0.0;
  }
  int32_t stack[kStack];
  int sp = 0;
  int32_t v = n > 1 ? 0 : ~0;
  for (;;) {
    if (v < 0) {
      const double* y = spos + int64_t(~v) * DIM;
      double dl[DIM], d2 = 0.0;
#pragma unroll
      for (int a = 0; a < DIM; ++a) {
        dl[a] = x[a] - __ldg(y + a);
        d2 = a == 0 ? dl[a] * dl[a] : fma(dl[a], dl[a], d2);
      }
      const double f = inv_d2(d2);
#pragma unroll
      for (int a = 0; a < DIM; ++a) acc[a] = fma(dl[a], f, acc[a]);
    } else {
      const double* r = rec + int64_t(v) * rec_len<DIM>();
      double diag2 = 0.0, rho2 = 0.0;
      bool point = true;
#pragma unroll
      for (int a = 0; a < DIM; ++a) {
        const double lo = __ldg(r + a), hi = __ldg(r + DIM + a);
        const double e = hi - lo;
        const double g = fmax(fmax(lo - x[a], x[a] - hi), 0.0);
        diag2 = a == 0 ? e * e : fma(e, e, diag2);
        rho2 = a == 0 ? g * g : fma(g, g, rho2);
        point = point && lo == hi;
      }
      // theta2 > 0: at theta = 0 a box whose squared diagonal underflows to 0 is still opened
      if (point || (theta2 > 0.0 && rho2 >= kMinD2 && diag2 <= theta2 * rho2)) {
        double dl[DIM], d2 = 0.0;
#pragma unroll
        for (int a = 0; a < DIM; ++a) {
          dl[a] = x[a] - __ldg(r + 2 * DIM + a);
          d2 = a == 0 ? dl[a] * dl[a] : fma(dl[a], dl[a], d2);
        }
        const double f = __ldg(r + 3 * DIM) * inv_d2(d2);
#pragma unroll
        for (int a = 0; a < DIM; ++a) acc[a] = fma(dl[a], f, acc[a]);
      } else {
        const int2 ch = __ldg(reinterpret_cast<const int2*>(r + 3 * DIM + 1));
        if (sp == kStack) {        // unreachable (depth <= 94, see the header); never a trap
          atomicExch(status, 1);
          break;
        }
        stack[sp++] = ch.y;
        v = ch.x;
        continue;
      }
    }
    if (sp == 0) break;
    v = stack[--sp];
  }
  const int64_t id = ids[s];
#pragma unroll
  for (int a = 0; a < DIM; ++a) partial[id * DIM + a] = k2 * acc[a];
}

// the caller's buffers of gsp_spring_bh_tree from the records
template <int DIM>
__global__ void bh_unpack_kernel(int64_t n, const double* __restrict__ rec,
                                 int32_t* __restrict__ children, int32_t* __restrict__ counts,
                                 double* __restrict__ boxes, double* __restrict__ centroids) {
  const int64_t v = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (v >= n - 1) return;
  const double* r = rec + v * rec_len<DIM>();
  const int2 ch = *reinterpret_cast<const int2*>(r + 3 * DIM + 1);
  children[2 * v] = ch.x;
  children[2 * v + 1] = ch.y;
  counts[v] = int32_t(r[3 * DIM]);
#pragma unroll
  for (int a = 0; a < DIM; ++a) {
    boxes[v * 2 * DIM + a] = r[a];
    boxes[v * 2 * DIM + DIM + a] = r[DIM + a];
    centroids[v * DIM + a] = r[2 * DIM + a];
  }
}

// The device scratch of one entry point, allocated once and reused by every tree built in it.
struct BhTree {
  int64_t n;
  int dim;
  cudaStream_t st;
  Scratch<uint64_t> keys, keys_sorted;
  Scratch<int32_t> ids, ids_sorted, parent, flags, status;
  Scratch<double> spos, rec, box;
  Scratch<char> cub_tmp;
  size_t cub_bytes = 0;

  BhTree(int64_t n_, int dim_, cudaStream_t st_)
      : n(n_), dim(dim_), st(st_), keys(st_), keys_sorted(st_), ids(st_), ids_sorted(st_),
        parent(st_), flags(st_), status(st_), spos(st_), rec(st_), box(st_), cub_tmp(st_) {}

  int sort(void* tmp, size_t& bytes) const {
    return (int)cub::DeviceRadixSort::SortPairs(tmp, bytes, keys.get(), keys_sorted.get(),
                                                ids.get(), ids_sorted.get(), (int)n, 0,
                                                kAxisBits * dim, st);
  }

  int alloc() {
    const size_t m = size_t(std::max<int64_t>(n - 1, 1));
    GSP_CUDA(keys.alloc(n));
    GSP_CUDA(keys_sorted.alloc(n));
    GSP_CUDA(ids.alloc(n));
    GSP_CUDA(ids_sorted.alloc(n));
    GSP_CUDA(parent.alloc(m + n));
    GSP_CUDA(flags.alloc(m));
    GSP_CUDA(status.alloc(1));
    GSP_CUDA(spos.alloc(size_t(n) * dim));
    GSP_CUDA(rec.alloc(m * (3 * dim + 2)));
    GSP_CUDA(box.alloc(kBoxBlocks * 2 * dim + 2 * dim));
    // CUB's two-phase protocol (as gsp::cub_temp), sized once for every sort of this call
    GSP_CUDA(cudaError_t(sort(nullptr, cub_bytes)));
    GSP_CUDA(cub_tmp.alloc(std::max<size_t>(cub_bytes, 16)));
    GSP_CUDA(cudaMemsetAsync(status.get(), 0, sizeof(int32_t), st));
    return GSP_OK;
  }

  template <int DIM>
  int build(const double* pos) {
    const unsigned g = (unsigned)ceil_div(n, 256);
    double* part = box.get() + 2 * DIM;
    bh_box_partial_kernel<DIM><<<kBoxBlocks, kBoxThreads, 0, st>>>(n, pos, part);
    GSP_LAUNCH_CHECK("bh_box_partial");
    bh_box_final_kernel<DIM><<<1, 32, 0, st>>>(kBoxBlocks, part, box.get());
    GSP_LAUNCH_CHECK("bh_box_final");
    bh_keys_kernel<DIM><<<g, 256, 0, st>>>(n, pos, box.get(), keys.get(), ids.get());
    GSP_LAUNCH_CHECK("bh_keys");
    size_t bytes = cub_bytes;
    GSP_CUDA(cudaError_t(sort(cub_tmp.get(), bytes)));
    bh_gather_kernel<DIM><<<g, 256, 0, st>>>(n, pos, ids_sorted.get(), spos.get(), flags.get());
    GSP_LAUNCH_CHECK("bh_gather");
    if (n > 1) {
      bh_build_kernel<DIM><<<g, 256, 0, st>>>(n, keys_sorted.get(), rec.get(), parent.get());
      GSP_LAUNCH_CHECK("bh_build");
      bh_aggregate_kernel<DIM><<<g, 256, 0, st>>>(n, spos.get(), rec.get(), parent.get(),
                                                  flags.get());
      GSP_LAUNCH_CHECK("bh_aggregate");
    }
    return GSP_OK;
  }

  template <int DIM>
  int walk(double theta, double k2, double* partial) {
    bh_walk_kernel<DIM><<<(unsigned)ceil_div(n, kWalkThreads), kWalkThreads, 0, st>>>(
        n, spos.get(), ids_sorted.get(), rec.get(), theta * theta, k2, partial, status.get());
    GSP_LAUNCH_CHECK("bh_walk");
    return GSP_OK;
  }

  // the walk's stack guard, read once at the end of the call
  int check_status() {
    int32_t h = 0;
    GSP_CUDA(cudaMemcpyAsync(&h, status.get(), sizeof(h), cudaMemcpyDeviceToHost, st));
    GSP_CUDA(cudaStreamSynchronize(st));
    if (h != 0) return fail(GSP_ERR_UNSUPPORTED, "Barnes-Hut walk stack exceeded");
    return GSP_OK;
  }
};

template <typename T>
int bh_step(BhTree& tree, const int32_t* indptr, const int32_t* indices, const T* data, double k,
            double t, double theta, const uint8_t* fixed, const double* pos_in, double* pos_out,
            double* partial) {
  const int64_t n = tree.n;
  int rc = GSP_OK;
  switch (tree.dim) {
    case 1: rc = tree.build<1>(pos_in); if (rc == GSP_OK) rc = tree.walk<1>(theta, k * k, partial); break;
    case 2: rc = tree.build<2>(pos_in); if (rc == GSP_OK) rc = tree.walk<2>(theta, k * k, partial); break;
    default: rc = tree.build<3>(pos_in); if (rc == GSP_OK) rc = tree.walk<3>(theta, k * k, partial); break;
  }
  if (rc != GSP_OK) return rc;
  spring::spring_update_kernel<T><<<(unsigned)ceil_div(n, 256), 256, 0, tree.st>>>(
      n, tree.dim, indptr, indices, data, k, t, fixed, 1, pos_in, partial, pos_out);
  GSP_LAUNCH_CHECK("spring_update");
  return GSP_OK;
}

#define GSP_REQUIRE_BH(n, dim, pos, theta)                                                      \
  GSP_REQUIRE((n) >= 0 && (n) < (int64_t(1) << 31), "bad vertex count");                        \
  GSP_REQUIRE((dim) >= 1 && (dim) <= 3, "Barnes-Hut layouts take dim 1, 2 or 3");               \
  GSP_REQUIRE(isfinite(theta) && (theta) >= 0.0, "theta must be finite and >= 0");              \
  GSP_REQUIRE((n) == 0 || (pos) != nullptr, "positions are NULL")

template <typename T>
int bh_step_api(int64_t n, int dim, const int32_t* indptr, const int32_t* indices, const T* data,
                double k, double t, const uint8_t* fixed, const double* pos_in, double* pos_out,
                double theta, cudaStream_t st) {
  GSP_REQUIRE_BH(n, dim, pos_in, theta);
  GSP_REQUIRE(n == 0 || (pos_out != nullptr && pos_out != pos_in),
              "pos_out must be a distinct block");
  if (n == 0) return GSP_OK;
  BhTree tree(n, dim, st);
  int rc = tree.alloc();
  if (rc != GSP_OK) return rc;
  Scratch<double> partial(st);
  GSP_CUDA(partial.alloc(size_t(n) * dim));
  rc = bh_step<T>(tree, indptr, indices, data, k, t, theta, fixed, pos_in, pos_out,
                  partial.get());
  return rc != GSP_OK ? rc : tree.check_status();
}

template <typename T>
int bh_layout(int64_t n, int dim, const int32_t* indptr, const int32_t* indices, const T* data,
              double k, int iterations, const double* temps_host, const uint8_t* fixed,
              double* pos, double* states, double theta, cudaStream_t st) {
  GSP_REQUIRE_BH(n, dim, pos, theta);
  GSP_REQUIRE(iterations >= 0, "iterations must be >= 0");
  GSP_REQUIRE(iterations == 0 || temps_host != nullptr, "temperatures are NULL");
  if (n == 0 || iterations == 0) return GSP_OK;
  const size_t block = size_t(n) * dim;
  BhTree tree(n, dim, st);
  int rc = tree.alloc();
  if (rc != GSP_OK) return rc;
  Scratch<double> partial(st);
  GSP_CUDA(partial.alloc(block));
  // with `states`, iteration it writes states[it]; otherwise pos and one scratch block alternate
  Scratch<double> other(st);
  if (states == nullptr) GSP_CUDA(other.alloc(block));
  const double* cur = pos;
  for (int it = 0; it < iterations; ++it) {
    double* next = states != nullptr ? states + it * block : (it % 2 == 0 ? other.get() : pos);
    rc = bh_step<T>(tree, indptr, indices, data, k, temps_host[it], theta, fixed, cur, next,
                    partial.get());
    if (rc != GSP_OK) return rc;
    cur = next;
  }
  if (cur != pos)
    GSP_CUDA(cudaMemcpyAsync(pos, cur, block * sizeof(double), cudaMemcpyDeviceToDevice, st));
  return tree.check_status();
}

int bh_tree_api(int64_t n, int dim, const double* pos, int32_t* ids, int32_t* children,
                int32_t* counts, double* boxes, double* centroids, cudaStream_t st) {
  GSP_REQUIRE_BH(n, dim, pos, 0.0);
  GSP_REQUIRE(n == 0 || ids != nullptr, "ids are NULL");
  GSP_REQUIRE(n <= 1 || (children != nullptr && counts != nullptr && boxes != nullptr &&
                         centroids != nullptr),
              "tree buffers are NULL");
  if (n == 0) return GSP_OK;
  BhTree tree(n, dim, st);
  int rc = tree.alloc();
  if (rc != GSP_OK) return rc;
  const unsigned g = (unsigned)ceil_div(n, 256);
  switch (dim) {
    case 1: rc = tree.build<1>(pos); break;
    case 2: rc = tree.build<2>(pos); break;
    default: rc = tree.build<3>(pos); break;
  }
  if (rc != GSP_OK) return rc;
  GSP_CUDA(cudaMemcpyAsync(ids, tree.ids_sorted.get(), n * sizeof(int32_t),
                           cudaMemcpyDeviceToDevice, st));
  if (n > 1) {
    switch (dim) {
      case 1: bh_unpack_kernel<1><<<g, 256, 0, st>>>(n, tree.rec.get(), children, counts, boxes, centroids); break;
      case 2: bh_unpack_kernel<2><<<g, 256, 0, st>>>(n, tree.rec.get(), children, counts, boxes, centroids); break;
      default: bh_unpack_kernel<3><<<g, 256, 0, st>>>(n, tree.rec.get(), children, counts, boxes, centroids); break;
    }
    GSP_LAUNCH_CHECK("bh_unpack");
  }
  return GSP_OK;
}

}  // namespace
}  // namespace gsp

extern "C" {

#define GSP_BH_API(SUF, T)                                                                      \
  int gsp_spring_step_bh_##SUF(int64_t n, int dim, const int32_t* indptr, const int32_t* indices, \
                               const T* data, double k, double t, const uint8_t* fixed,         \
                               const double* pos_in, double* pos_out, double theta,             \
                               void* stream) {                                                  \
    return gsp::bh_step_api<T>(n, dim, indptr, indices, data, k, t, fixed, pos_in, pos_out,    \
                               theta, gsp::as_stream(stream));                                  \
  }                                                                                             \
  int gsp_spring_layout_bh_##SUF(int64_t n, int dim, const int32_t* indptr,                     \
                                 const int32_t* indices, const T* data, double k,               \
                                 int iterations, const double* temps_host,                      \
                                 const uint8_t* fixed, double* pos, double* states,             \
                                 double theta, void* stream) {                                  \
    return gsp::bh_layout<T>(n, dim, indptr, indices, data, k, iterations, temps_host, fixed,  \
                             pos, states, theta, gsp::as_stream(stream));                       \
  }

GSP_BH_API(f32, float)
GSP_BH_API(f64, double)

int gsp_spring_bh_tree(int64_t n, int dim, const double* pos, int32_t* ids, int32_t* children,
                       int32_t* counts, double* boxes, double* centroids, void* stream) {
  return gsp::bh_tree_api(n, dim, pos, ids, children, counts, boxes, centroids,
                          gsp::as_stream(stream));
}

}  // extern "C"
