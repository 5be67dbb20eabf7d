// Conjugate gradients on (diag(a) * tau * L + diag(d)) X = B for a block of right-hand sides.
//
// Replaces scipy.sparse.linalg.cg on the LinearOperator of
// pygsp/learning.py:326-337 (regression_tikhonov, tau > 0: x -> M x + tau L x, one solve per
// column in a Python loop) and the sparse direct solve of the constrained problem
// (:350-365, as CG on L restricted to the unlabelled vertices).  All columns advance
// together: the product with L is the SpMM step kernel of the filter path, the vector
// updates are fused with their dot products, every per-column scalar stays on the device,
// and reductions are two-level in a fixed order (bit-reproducible): per-CTA partials, added over
// the CTAs in order by sum_parts (csrc/reduce.cuh) or by load_totals.
//
//   spmm      Q = tau L P                                   (cheby_step, FIRST form, no r)
//   apply     Q = a.Q + d.P ; partial sums of P.Q per column
//   update    alpha = rr/pq ; X += alpha P ; R -= alpha Q ; partial sums of R.R
//   direction beta = rr'/rr ; P = R + beta P ; rr history[it+1] = rr'
#include "reduce.cuh"
#include "step.cuh"

namespace gsp {

constexpr int kCgThreads = 256;
constexpr int kCgMaxBlocks = 1024;

// per-column sum over the block of `v` (threads with the same column c = t % cw), result to
// out[c]; fixed order.
__device__ __forceinline__ void block_colsum(double v, int cw, int nsig, double* out) {
  __shared__ double sh[kCgThreads];
  sh[threadIdx.x] = v;
  __syncthreads();
  if (threadIdx.x < cw && int(threadIdx.x) < nsig) {
    double acc = 0;
    for (int k = threadIdx.x; k < kCgThreads; k += cw) acc += sh[k];
    out[threadIdx.x] = acc;
  }
  __syncthreads();
}

// total[c] = sum over `parts` partial rows, into shared memory (every block recomputes it)
__device__ __forceinline__ void load_totals(const double* part, int parts, int nsig, double* sh_tot) {
  if (int(threadIdx.x) < nsig) {
    double acc = 0;
    for (int b = 0; b < parts; ++b) acc += part[int64_t(b) * nsig + threadIdx.x];
    sh_tot[threadIdx.x] = acc;
  }
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(kCgThreads)
cg_init_kernel(int64_t n, int nsig, int cw, const T* __restrict__ B, T* __restrict__ X,
               T* __restrict__ R, T* __restrict__ P, double* part_rr) {
  const int c = threadIdx.x % cw, rl = threadIdx.x / cw, rpb = kCgThreads / cw;
  double acc = 0;
  if (c < nsig)
    for (int64_t row = int64_t(blockIdx.x) * rpb + rl; row < n; row += int64_t(gridDim.x) * rpb) {
      const int64_t i = row * nsig + c;
      const T b = B[i];
      X[i] = T(0);
      R[i] = b;
      P[i] = b;
      acc += double(b) * double(b);
    }
  block_colsum(acc, cw, nsig, part_rr + int64_t(blockIdx.x) * nsig);
}

template <typename T>
__global__ void __launch_bounds__(kCgThreads)
cg_apply_kernel(int64_t n, int nsig, int cw, const T* __restrict__ a_row, const T* __restrict__ d_row,
                const T* __restrict__ P, T* __restrict__ Q, double* part_pq) {
  const int c = threadIdx.x % cw, rl = threadIdx.x / cw, rpb = kCgThreads / cw;
  double acc = 0;
  if (c < nsig)
    for (int64_t row = int64_t(blockIdx.x) * rpb + rl; row < n; row += int64_t(gridDim.x) * rpb) {
      const int64_t i = row * nsig + c;
      const double p = double(P[i]);
      double q = double(Q[i]);
      if (a_row) q *= double(a_row[row]);
      if (d_row) q += double(d_row[row]) * p;
      const T qs = T(q);
      Q[i] = qs;
      acc += p * double(qs);
    }
  block_colsum(acc, cw, nsig, part_pq + int64_t(blockIdx.x) * nsig);
}

template <typename T>
__global__ void __launch_bounds__(kCgThreads)
cg_update_kernel(int64_t n, int nsig, int cw, T* __restrict__ X, T* __restrict__ R,
                 const T* __restrict__ P, const T* __restrict__ Q, const double* rr_cur,
                 const double* part_pq, int parts, double* part_rr) {
  __shared__ double pq[kCgThreads];
  load_totals(part_pq, parts, nsig, pq);
  const int c = threadIdx.x % cw, rl = threadIdx.x / cw, rpb = kCgThreads / cw;
  double acc = 0;
  if (c < nsig) {
    const double den = pq[c];
    const double alpha = den > 0 ? rr_cur[c] / den : 0.0;      // a converged column stays put
    for (int64_t row = int64_t(blockIdx.x) * rpb + rl; row < n; row += int64_t(gridDim.x) * rpb) {
      const int64_t i = row * nsig + c;
      X[i] = T(double(X[i]) + alpha * double(P[i]));
      const T r = T(double(R[i]) - alpha * double(Q[i]));
      R[i] = r;
      acc += double(r) * double(r);
    }
  }
  block_colsum(acc, cw, nsig, part_rr + int64_t(blockIdx.x) * nsig);
}

template <typename T>
__global__ void __launch_bounds__(kCgThreads)
cg_direction_kernel(int64_t n, int nsig, int cw, const T* __restrict__ R, T* __restrict__ P,
                    const double* rr_cur, const double* part_rr, int parts, double* rr_next) {
  __shared__ double rn[kCgThreads];
  load_totals(part_rr, parts, nsig, rn);
  const int c = threadIdx.x % cw, rl = threadIdx.x / cw, rpb = kCgThreads / cw;
  if (blockIdx.x == 0 && int(threadIdx.x) < nsig) rr_next[threadIdx.x] = rn[threadIdx.x];
  if (c < nsig) {
    const double beta = rr_cur[c] > 0 ? rn[c] / rr_cur[c] : 0.0;
    for (int64_t row = int64_t(blockIdx.x) * rpb + rl; row < n; row += int64_t(gridDim.x) * rpb) {
      const int64_t i = row * nsig + c;
      P[i] = T(double(R[i]) + beta * double(P[i]));
    }
  }
}

// Iterations [it0, it1).  scal = rr[(cap+1) x nsig] | part_pq[kCgMaxBlocks x nsig] |
// part_rr[kCgMaxBlocks x nsig] (doubles).  it0 == 0 starts from X = 0: R = P = B.
template <typename T>
int cg_run(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices, const T* data,
           double tau, const T* a_row, const T* d_row, const T* B, T* X, T* R, T* P, T* Q, int nsig,
           int it0, int it1, int cap, double* scal, cudaStream_t st) {
  GSP_REQUIRE(n >= 1 && nsig >= 1 && nsig <= kCgThreads, "block CG: 1..256 right-hand sides per call");
  GSP_REQUIRE(it0 >= 0 && it0 <= it1 && it1 <= cap, "bad iteration range");
  int cw = 1;                                      // columns per block pass: a power of two >= nsig
  while (cw < nsig) cw *= 2;
  const int blocks = pass_blocks(n, kCgThreads / cw, kCgMaxBlocks);
  double* rr = scal;
  double* part_pq = scal + int64_t(cap + 1) * nsig;
  double* part_rr = part_pq + int64_t(kCgMaxBlocks) * nsig;
  if (it0 == 0) {
    cg_init_kernel<T><<<blocks, kCgThreads, 0, st>>>(n, nsig, cw, B, X, R, P, part_rr);
    GSP_LAUNCH_CHECK("cg_init");
    const int rc = sum_parts(part_rr, blocks, nsig, rr, st);
    if (rc != GSP_OK) return rc;
  }
  Step<T> spmm{nnz, indptr, indices, data};       // Q = tau L P: the first form, no r_i
  spmm.x_cur = P;
  spmm.x_new = spmm.r = Q;
  spmm.r_rows = n;
  spmm.nsig = nsig;
  spmm.first = true;
  spmm.alpha = tau;
  for (int it = it0; it < it1; ++it) {
    int rc = run_step<T>(spmm, 0, n, nullptr, nullptr, st);
    if (rc != GSP_OK) return rc;
    cg_apply_kernel<T><<<blocks, kCgThreads, 0, st>>>(n, nsig, cw, a_row, d_row, P, Q, part_pq);
    cg_update_kernel<T><<<blocks, kCgThreads, 0, st>>>(n, nsig, cw, X, R, P, Q,
                                                       rr + int64_t(it) * nsig, part_pq, blocks,
                                                       part_rr);
    cg_direction_kernel<T><<<blocks, kCgThreads, 0, st>>>(n, nsig, cw, R, P,
                                                          rr + int64_t(it) * nsig, part_rr,
                                                          blocks, rr + int64_t(it + 1) * nsig);
    note_launch(2);
    GSP_LAUNCH_CHECK("cg_iteration");
  }
  return GSP_OK;
}

}  // namespace gsp

extern "C" {
#define GSP_CG_API(SUF, T)                                                                        \
  int gsp_cg_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,        \
                   const T* data, double tau, const T* row_scale, const T* diag, const T* B, T* X, \
                   T* R, T* P, T* Q, int64_t nsig, int it0, int it1, int cap, double* scal_dev,  \
                   void* stream) {                                                                \
    return gsp::cg_run<T>(n, nnz, indptr, indices, data, tau, row_scale, diag, B, X, R, P, Q,     \
                          (int)nsig, it0, it1, cap, scal_dev, gsp::as_stream(stream));            \
  }
GSP_CG_API(f32, float)
GSP_CG_API(f64, double)
}
