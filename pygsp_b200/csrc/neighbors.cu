// Exhaustive nearest-neighbour search in any dimension and the symmetrisations of
// NNGraph (SURVEY.md 8f-4, DESIGN.md 4.13).
//
//   * k nearest neighbours (self excluded by index) for the Minkowski metrics p = 1, 2, inf and
//     any p >= 1 -- the KDTree(X).query(X, k + 1, p) of pygsp/graphs/nngraphs/nngraph.py:213-216
//     for point clouds of any dimension (image patches, embeddings), where a cell grid
//     (generate.cu) does not apply;
//   * the radius graph {j != i : dist(x_i, x_j) <= epsilon} -- query_ball_point and the self
//     filter of nngraph.py:228-283 -- as count / scan / fill, rows sorted by column;
//   * utils.symmetrize(W, 'maximum' | 'fill' | 'tril' | 'triu') (utils.py:244-277) as a merge of
//     the rows of W and W^T ('average' is csr_average in graph.cu).
//
// Search tiling: a CTA owns kQ query rows and streams the whole cloud through shared memory in
// tiles of kC candidates x kS dimensions (query and candidate slabs double-buffered with
// cp.async).  Each of the 256 threads keeps a 4 x 4 block of partial distances in registers
// across the slabs of one candidate tile, so any dimension works and the sum runs in dimension
// order (zero padding adds exact zeros).  The finished 64 x 64 tile goes to shared memory and
// thread q (< kQ) merges row q into its query's sorted list of k best (accumulated distance,
// id) pairs: candidates arrive in increasing id, so a candidate enters only if it is strictly
// closer than the current k-th, and the list is the (distance, id) order whatever the tiling.
// Comparisons run on the accumulated value (sum |d|, sum d^2, max |d|, sum |d|^p), as
// cKDTree does; the root is taken once per kept pair.  All arithmetic is double.
#include <cub/cub.cuh>
#include <math.h>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {
namespace {

constexpr int kQ = 64;            // query rows per CTA
constexpr int kC = 64;            // candidate points per tile
constexpr int kS = 16;            // dimensions per slab
constexpr int kLd = kS + 1;       // padded slab row: column reads by 16 rows hit 16 bank pairs
constexpr int kDLd = kC + 1;      // padded row of the distance tile
constexpr int kMaxNbK = 32;       // = kMaxK of generate.cu: gsp_knn_to_csr_* takes the output
constexpr int kLs = kMaxNbK + 1;  // padded row of the per-query lists
constexpr int kNbThreads = 256;

enum Metric { kL1 = 0, kL2 = 1, kLinf = 2, kLp = 3 };
enum Mode { kKnn = 0, kCount = 1, kFill = 2 };

constexpr size_t kSmemBytes =
    sizeof(double) * (2 * kQ * kLd + 2 * kC * kLd + kQ * kDLd + kQ * kLs) + sizeof(int) * kQ * kLs;

template <int M>
__device__ __forceinline__ double accumulate(double acc, double diff, double p) {
  if (M == kL1) return acc + fabs(diff);
  if (M == kL2) return fma(diff, diff, acc);
  if (M == kLinf) return fmax(acc, fabs(diff));
  return acc + pow(fabs(diff), p);
}

template <int M>
__device__ __forceinline__ double finish(double acc, double p) {
  if (M == kL2) return sqrt(acc);
  if (M == kLp) return pow(acc, 1.0 / p);
  return acc;
}

// 8-byte cp.async; src_bytes = 0 writes a zero (rows / dimensions past the cloud)
__device__ __forceinline__ void copy8(double* dst, const double* src, bool valid) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(s), "l"(src),
               "r"(valid ? 8 : 0));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// MODE kKnn:   out_idx / out_dist are the (n, k) lists.
// MODE kCount: indptr[i + 1] = row size.
// MODE kFill:  row i is written at indptr[i] into out_idx / out_dist, in column order.
// SEG: query i only sees the candidates of its segment [seg_start[s], seg_start[s + 1]),
// s = seg_id[i].  The CTA walks the candidate tiles covering the segments of its first and last
// query only, and each query skips the columns of a tile outside its own segment -- the same
// per-pair test, in the same (tile, column) order, as the unsegmented search of the segment.
template <int M, int MODE, bool SEG>
__device__ __forceinline__ void neighbors_body(int64_t n, int d, const double* __restrict__ pts,
                                               int k, double p, double eps_acc, int32_t* indptr,
                                               int32_t* out_idx, double* out_dist,
                                               const int64_t* __restrict__ seg_start,
                                               const int32_t* __restrict__ seg_id) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* sq = reinterpret_cast<double*>(smem_raw);   // [2][kQ][kLd]
  double* sc = sq + 2 * kQ * kLd;                     // [2][kC][kLd]
  double* sdist = sc + 2 * kC * kLd;                  // [kQ][kDLd]
  double* bd = sdist + kQ * kDLd;                     // [kQ][kLs]
  int* bi = reinterpret_cast<int*>(bd + kQ * kLs);    // [kQ][kLs]

  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t q0 = int64_t(blockIdx.x) * kQ;
  const int nslab = (d + kS - 1) / kS;
  int64_t t0 = 0, ntile = (n + kC - 1) / kC;
  int64_t seg_lo = 0, seg_hi = n;     // candidate range of this thread's query (SEG)
  if (SEG) {
    const int64_t qlast = (q0 + kQ < n ? q0 + kQ : n) - 1;
    const int64_t c_lo = __ldg(seg_start + __ldg(seg_id + q0));
    const int64_t c_hi = __ldg(seg_start + __ldg(seg_id + qlast) + 1);
    t0 = c_lo / kC;
    ntile = c_hi > c_lo ? (c_hi + kC - 1) / kC - t0 : 0;
    if (tid < kQ && q0 + tid < n) {
      const int s = __ldg(seg_id + q0 + tid);
      seg_lo = __ldg(seg_start + s);
      seg_hi = __ldg(seg_start + s + 1);
    }
  }
  const int64_t nstep = ntile * nslab;

  auto load = [&](int64_t step, int buf) {
    const int64_t t = t0 + step / nslab;
    const int dim0 = int(step - (t - t0) * nslab) * kS;
    double* dq = sq + buf * kQ * kLd;
    double* dc = sc + buf * kC * kLd;
    for (int e = tid; e < kQ * kS; e += kNbThreads) {
      const int r = e / kS, s = e - r * kS, dim = dim0 + s;
      const int64_t qi = q0 + r, ci = t * kC + r;
      const bool qv = qi < n && dim < d, cv = ci < n && dim < d;
      copy8(dq + r * kLd + s, qv ? pts + qi * d + dim : pts, qv);
      copy8(dc + r * kLd + s, cv ? pts + ci * d + dim : pts, cv);
    }
    cp_commit();
  };

  // selection state of thread q = tid < kQ (one thread owns one query's list)
  const int64_t my_q = q0 + tid;
  const bool selector = tid < kQ && my_q < n;
  double thr = INFINITY;     // k-th best accumulated distance once the list is full
  int found = 0;
  int64_t cnt = 0;
  int64_t o = (MODE == kFill && selector) ? indptr[my_q] : 0;

  double acc[4][4];
  if (!SEG || nstep > 0) load(0, 0);
  for (int64_t step = 0; step < nstep; ++step) {
    const int buf = int(step & 1);
    if (step + 1 < nstep) {
      load(step + 1, buf ^ 1);
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    const int64_t t = t0 + step / nslab;
    const int sl = int(step - (t - t0) * nslab);
    if (sl == 0) {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    }
    const double* cq = sq + buf * kQ * kLd;
    const double* cc = sc + buf * kC * kLd;
#pragma unroll 4
    for (int s = 0; s < kS; ++s) {
      double qv[4], cv[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) qv[i] = cq[(ty + 16 * i) * kLd + s];
#pragma unroll
      for (int j = 0; j < 4; ++j) cv[j] = cc[(tx + 16 * j) * kLd + s];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = accumulate<M>(acc[i][j], qv[i] - cv[j], p);
    }
    if (sl == nslab - 1) {     // tile finished: hand it to the selecting threads
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) sdist[(ty + 16 * i) * kDLd + tx + 16 * j] = acc[i][j];
      __syncthreads();
      if (selector) {
        const int64_t c0 = t * kC;
        const int cn = n - c0 < kC ? int(n - c0) : kC;
        const double* row = sdist + tid * kDLd;
        int cb = 0, ce = cn;
        if (SEG) {
          cb = seg_lo > c0 ? int(seg_lo - c0 < kC ? seg_lo - c0 : kC) : 0;
          ce = seg_hi - c0 < cn ? int(seg_hi - c0 > 0 ? seg_hi - c0 : 0) : cn;
        }
        for (int c = cb; c < ce; ++c) {
          const int64_t cand = c0 + c;
          if (cand == my_q) continue;
          const double a = row[c];
          if (MODE == kKnn) {
            if (!(a < thr)) continue;
            double* ld = bd + tid * kLs;
            int* li = bi + tid * kLs;
            int pos = found < k ? found : k - 1;
            while (pos > 0 && ld[pos - 1] > a) {   // equal keys keep the smaller id first
              ld[pos] = ld[pos - 1];
              li[pos] = li[pos - 1];
              --pos;
            }
            ld[pos] = a;
            li[pos] = int(cand);
            if (found < k) ++found;
            if (found == k) thr = ld[k - 1];
          } else if (a <= eps_acc) {
            if (MODE == kFill) {
              out_idx[o] = int32_t(cand);
              out_dist[o] = finish<M>(a, p);
              ++o;
            } else {
              ++cnt;
            }
          }
        }
      }
    }
    __syncthreads();           // buffer `buf` and the distance tile are free again
  }

  if (!selector) return;
  if (MODE == kKnn) {
    const double* ld = bd + tid * kLs;
    const int* li = bi + tid * kLs;
    for (int j = 0; j < k; ++j) {
      out_idx[my_q * k + j] = j < found ? li[j] : -1;
      out_dist[my_q * k + j] = j < found ? finish<M>(ld[j], p) : 0.0;
    }
  } else if (MODE == kCount) {
    if (my_q == 0) indptr[0] = 0;
    indptr[my_q + 1] = int32_t(cnt);
  }
}

template <int M, int MODE>
__global__ void __launch_bounds__(kNbThreads, 2)
    neighbors_kernel(int64_t n, int d, const double* __restrict__ pts, int k, double p,
                     double eps_acc, int32_t* indptr, int32_t* out_idx, double* out_dist) {
  neighbors_body<M, MODE, false>(n, d, pts, k, p, eps_acc, indptr, out_idx, out_dist, nullptr,
                                 nullptr);
}

template <int M, int MODE>
__global__ void __launch_bounds__(kNbThreads, 2)
    neighbors_seg_kernel(int64_t n, int d, const double* __restrict__ pts, int k, double p,
                         double eps_acc, int32_t* indptr, int32_t* out_idx, double* out_dist,
                         const int64_t* __restrict__ seg_start,
                         const int32_t* __restrict__ seg_id) {
  neighbors_body<M, MODE, true>(n, d, pts, k, p, eps_acc, indptr, out_idx, out_dist, seg_start,
                                seg_id);
}

// seg_start == nullptr: the whole cloud; otherwise the segmented search (seg_id per vertex)
template <int MODE>
int launch_neighbors(int64_t n, int d, const double* pts, int k, double p, double eps_acc,
                     int32_t* indptr, int32_t* out_idx, double* out_dist, cudaStream_t st,
                     const int64_t* seg_start = nullptr, const int32_t* seg_id = nullptr) {
  const int blocks = (int)ceil_div(n, kQ);
#define GSP_NB_LAUNCH(M)                                                                        \
  do {                                                                                          \
    if (seg_start == nullptr) {                                                                 \
      auto kern = neighbors_kernel<M, MODE>;                                                    \
      GSP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                                    (int)kSmemBytes));                                          \
      kern<<<blocks, kNbThreads, kSmemBytes, st>>>(n, d, pts, k, p, eps_acc, indptr, out_idx,   \
                                                   out_dist);                                   \
    } else {                                                                                    \
      auto kern = neighbors_seg_kernel<M, MODE>;                                                \
      GSP_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,          \
                                    (int)kSmemBytes));                                          \
      kern<<<blocks, kNbThreads, kSmemBytes, st>>>(n, d, pts, k, p, eps_acc, indptr, out_idx,   \
                                                   out_dist, seg_start, seg_id);                \
    }                                                                                           \
  } while (0)
  if (p == 1.0) GSP_NB_LAUNCH(kL1);
  else if (p == 2.0) GSP_NB_LAUNCH(kL2);
  else if (isinf(p)) GSP_NB_LAUNCH(kLinf);
  else GSP_NB_LAUNCH(kLp);
#undef GSP_NB_LAUNCH
  GSP_LAUNCH_CHECK("neighbors");
  return GSP_OK;
}

// the radius test on the accumulated value, as cKDTree compares (sum |d|^p <= eps^p)
double radius_key(double eps, double p) {
  if (p == 2.0) return eps * eps;
  if (p == 1.0 || isinf(p)) return eps;
  return pow(eps, p);
}

// ---- utils.symmetrize (utils.py:244-277) as a merge of row i of A = W and B = W^T ---------
enum SymMode { kSymMaximum = 0, kSymFill = 1, kSymTril = 2, kSymTriu = 3 };

template <typename T, bool FILL>
__global__ void csr_symmetrize_kernel(int64_t n, int mode, const int32_t* __restrict__ a_ptr,
                                      const int32_t* __restrict__ a_idx,
                                      const T* __restrict__ a_val,
                                      const int32_t* __restrict__ b_ptr,
                                      const int32_t* __restrict__ b_idx,
                                      const T* __restrict__ b_val, int32_t* s_ptr,
                                      int32_t* s_idx, T* s_val) {
  const int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (!FILL && row == 0) s_ptr[0] = 0;
  if (row >= n) return;
  int ia = a_ptr[row], ea = a_ptr[row + 1], ib = b_ptr[row], eb = b_ptr[row + 1];
  int o = FILL ? s_ptr[row] : 0;
  while (ia < ea || ib < eb) {
    const int ca = ia < ea ? a_idx[ia] : INT_MAX;
    const int cb = ib < eb ? b_idx[ib] : INT_MAX;
    const int col = min(ca, cb);
    T a = T(0), b = T(0);            // a = W[row, col], b = W[col, row]
    if (ca == col) a = a_val[ia++];
    if (cb == col) b = b_val[ib++];
    T v;
    if (mode == kSymFill) {
      // W2 = W + ((A + A^T) - A) o W^T with A = W > 0, then (W2 + W2^T) / 2
      const T w_rc = a + ((!(a > T(0)) && b > T(0)) ? b : T(0));
      const T w_cr = b + ((!(b > T(0)) && a > T(0)) ? a : T(0));
      const T sum = w_rc + w_cr;
      v = sum / T(2);
      if (sum == T(0)) v = T(0);
    } else {
      if (mode == kSymTril) {        // sparse.tril: entries with col <= row
        if (col > row) a = T(0);
        if (row > col) b = T(0);
      } else if (mode == kSymTriu) {
        if (col < row) a = T(0);
        if (row < col) b = T(0);
      }
      // W - W o [W^T > W] + W^T o [W^T > W]
      v = b > a ? b : a;
    }
    if (v != T(0)) {
      if (FILL) { s_idx[o] = col; s_val[o] = v; }
      ++o;
    }
  }
  if (!FILL) s_ptr[row + 1] = o;
}

template <typename T>
int csr_symmetrize(bool fill, int64_t n, int mode, const int32_t* ap, const int32_t* ai,
                   const T* ad, const int32_t* bp, const int32_t* bi, const T* bd, int32_t* sp,
                   int32_t* si, T* sd, int64_t* nnz, cudaStream_t st) {
  GSP_REQUIRE(mode >= kSymMaximum && mode <= kSymTriu, "unknown symmetrisation mode");
  const int blocks = (int)ceil_div(n > 0 ? n : 1, 256);
  if (fill) {
    if (n == 0) return GSP_OK;
    csr_symmetrize_kernel<T, true><<<blocks, 256, 0, st>>>(n, mode, ap, ai, ad, bp, bi, bd, sp, si,
                                                           sd);
    GSP_LAUNCH_CHECK("csr_symmetrize_fill");
    return GSP_OK;
  }
  csr_symmetrize_kernel<T, false><<<blocks, 256, 0, st>>>(n, mode, ap, ai, ad, bp, bi, bd, sp,
                                                          nullptr, nullptr);
  GSP_LAUNCH_CHECK("csr_symmetrize_count");
  return scan_rows(sp, n, nnz, st);
}

// w = exp(-d^2 / sigma), the weights of nngraph.py:221-226, 276-281
template <typename T>
__global__ void gauss_weights_kernel(int64_t nnz, const double* __restrict__ dist, double sigma,
                                     T* w) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= nnz) return;
  const double x = dist[e];
  w[e] = T(exp(-(x * x) / sigma));
}

template <typename T>
int gauss_weights(int64_t nnz, const double* dist, double sigma, T* w, cudaStream_t st) {
  if (nnz == 0) return GSP_OK;
  gauss_weights_kernel<T><<<(int)ceil_div(nnz, 256), 256, 0, st>>>(nnz, dist, sigma, w);
  GSP_LAUNCH_CHECK("gauss_weights");
  return GSP_OK;
}

}  // namespace
}  // namespace gsp

#define GSP_REQUIRE_CLOUD(n, d, p)                                                              \
  GSP_REQUIRE((n) >= 1 && (n) < (int64_t(1) << 31) && (d) >= 1, "bad point cloud");            \
  GSP_REQUIRE((p) >= 1.0, "Minkowski order p must be >= 1")

extern "C" {

int gsp_knn_brute(int64_t n, int d, const double* points, int k, double p, int32_t* nn_idx,
                  double* nn_dist, void* stream) {
  GSP_REQUIRE_CLOUD(n, d, p);
  GSP_REQUIRE(k >= 1 && k <= gsp::kMaxNbK && k < n, "k must be in [1, 32] and < n");
  return gsp::launch_neighbors<gsp::kKnn>(n, d, points, k, p, 0.0, nullptr, nn_idx, nn_dist,
                                          gsp::as_stream(stream));
}

int gsp_radius_count(int64_t n, int d, const double* points, double epsilon, double p,
                     int32_t* indptr, int64_t* nnz, void* stream) {
  GSP_REQUIRE_CLOUD(n, d, p);
  GSP_REQUIRE(epsilon >= 0, "epsilon must be >= 0");
  cudaStream_t st = gsp::as_stream(stream);
  const int rc = gsp::launch_neighbors<gsp::kCount>(
      n, d, points, 1, p, gsp::radius_key(epsilon, p), indptr, nullptr, nullptr, st);
  if (rc != GSP_OK) return rc;
  return gsp::scan_rows(indptr, n, nnz, st);
}

int gsp_radius_fill_f64(int64_t n, int d, const double* points, double epsilon, double p,
                        const int32_t* indptr, int32_t* indices, double* dist, void* stream) {
  GSP_REQUIRE_CLOUD(n, d, p);
  GSP_REQUIRE(epsilon >= 0, "epsilon must be >= 0");
  return gsp::launch_neighbors<gsp::kFill>(n, d, points, 1, p, gsp::radius_key(epsilon, p),
                                           const_cast<int32_t*>(indptr), indices, dist,
                                           gsp::as_stream(stream));
}

#define GSP_REQUIRE_SEGMENTS(n_seg, seg_start, seg_id)                                         \
  GSP_REQUIRE((n_seg) >= 1 && (seg_start) && (seg_id), "bad segment table")

int gsp_knn_brute_seg(int64_t n, int d, const double* points, int k, double p, int64_t n_seg,
                      const int64_t* seg_start, const int32_t* seg_id, int32_t* nn_idx,
                      double* nn_dist, void* stream) {
  GSP_REQUIRE_CLOUD(n, d, p);
  GSP_REQUIRE_SEGMENTS(n_seg, seg_start, seg_id);
  GSP_REQUIRE(k >= 1 && k <= gsp::kMaxNbK, "k must be in [1, 32]");
  return gsp::launch_neighbors<gsp::kKnn>(n, d, points, k, p, 0.0, nullptr, nn_idx, nn_dist,
                                          gsp::as_stream(stream), seg_start, seg_id);
}

int gsp_radius_count_seg(int64_t n, int d, const double* points, double epsilon, double p,
                         int64_t n_seg, const int64_t* seg_start, const int32_t* seg_id,
                         int32_t* indptr, int64_t* nnz, void* stream) {
  GSP_REQUIRE_CLOUD(n, d, p);
  GSP_REQUIRE_SEGMENTS(n_seg, seg_start, seg_id);
  GSP_REQUIRE(epsilon >= 0, "epsilon must be >= 0");
  cudaStream_t st = gsp::as_stream(stream);
  const int rc = gsp::launch_neighbors<gsp::kCount>(n, d, points, 1, p,
                                                    gsp::radius_key(epsilon, p), indptr, nullptr,
                                                    nullptr, st, seg_start, seg_id);
  if (rc != GSP_OK) return rc;
  return gsp::scan_rows(indptr, n, nnz, st);
}

int gsp_radius_fill_seg_f64(int64_t n, int d, const double* points, double epsilon, double p,
                            int64_t n_seg, const int64_t* seg_start, const int32_t* seg_id,
                            const int32_t* indptr, int32_t* indices, double* dist,
                            void* stream) {
  GSP_REQUIRE_CLOUD(n, d, p);
  GSP_REQUIRE_SEGMENTS(n_seg, seg_start, seg_id);
  GSP_REQUIRE(epsilon >= 0, "epsilon must be >= 0");
  return gsp::launch_neighbors<gsp::kFill>(n, d, points, 1, p, gsp::radius_key(epsilon, p),
                                           const_cast<int32_t*>(indptr), indices, dist,
                                           gsp::as_stream(stream), seg_start, seg_id);
}

#define GSP_NEIGHBOR_API(SUF, T)                                                                \
  int gsp_csr_symmetrize_count_##SUF(int64_t n, int mode, const int32_t* a_indptr,              \
                                     const int32_t* a_indices, const T* a_data,                 \
                                     const int32_t* b_indptr, const int32_t* b_indices,         \
                                     const T* b_data, int32_t* s_indptr, int64_t* nnz,          \
                                     void* stream) {                                            \
    return gsp::csr_symmetrize<T>(false, n, mode, a_indptr, a_indices, a_data, b_indptr,        \
                                  b_indices, b_data, s_indptr, nullptr, nullptr, nnz,           \
                                  gsp::as_stream(stream));                                      \
  }                                                                                             \
  int gsp_csr_symmetrize_fill_##SUF(int64_t n, int mode, const int32_t* a_indptr,               \
                                    const int32_t* a_indices, const T* a_data,                  \
                                    const int32_t* b_indptr, const int32_t* b_indices,          \
                                    const T* b_data, const int32_t* s_indptr,                   \
                                    int32_t* s_indices, T* s_data, void* stream) {              \
    return gsp::csr_symmetrize<T>(true, n, mode, a_indptr, a_indices, a_data, b_indptr,         \
                                  b_indices, b_data, const_cast<int32_t*>(s_indptr),            \
                                  s_indices, s_data, nullptr, gsp::as_stream(stream));          \
  }                                                                                             \
  int gsp_gauss_weights_##SUF(int64_t nnz, const double* dist, double sigma, T* w,              \
                              void* stream) {                                                   \
    return gsp::gauss_weights<T>(nnz, dist, sigma, w, gsp::as_stream(stream));                  \
  }

GSP_NEIGHBOR_API(f32, float)
GSP_NEIGHBOR_API(f64, double)

}  // extern "C"
