// Per-signal Krylov bases of Lanczos filtering (pygsp_b200/filters/approximations.py).
//
// Replaces, for pygsp/filters/approximations.py:
//   * lanczos(A, order, x) (:281-341): one Lanczos process per signal column with full
//     reorthogonalisation, in the reference's step order                  -> gsp_krylov_basis_*
//   * the combination V Q f(Theta) Q^T V^T s of lanczos_op (:266-276)     -> gsp_krylov_combine_*
//
// The basis is one (order + 1, n, nsig) allocation: vector k of every column is the (n, nsig)
// row-major block V[k], so the SpMM (csrc/cheby.cu) takes a slice of it directly.  Slot k + 1
// is the residual r of step k until it is normalised into q_{k+1}.
//
// Columns never mix.  Every reduction over rows is the two-level column reduction of
// csrc/reduce.cuh, in double also for float blocks, so a column's bits do not depend on nsig, on
// the other columns, or on how the columns are chunked.
#include <cfloat>

#include "reduce.cuh"

namespace gsp {
namespace {

// r = A q through the SpMM of csrc/cheby.cu
inline int spmm(int64_t n, const int32_t* indptr, const int32_t* indices, const float* data,
                const float* x, int64_t ns, float* y, cudaStream_t st) {
  return gsp_spmm_f32(n, indptr, indices, data, x, ns, y, st);
}
inline int spmm(int64_t n, const int32_t* indptr, const int32_t* indices, const double* data,
                const double* x, int64_t ns, double* y, cudaStream_t st) {
  return gsp_spmm_f64(n, indptr, indices, data, x, ns, y, st);
}

constexpr int kGramTile = 8;           // basis vectors per CTA of the per-column Gram
constexpr int kFilterTile = 16;        // filters per pass of the combine over V
constexpr double kBreakdown = 16.0;    // breakdown threshold, in units of the dtype's epsilon

template <typename T> struct Eps;
template <> struct Eps<float> { static constexpr double value = FLT_EPSILON; };
template <> struct Eps<double> { static constexpr double value = DBL_EPSILON; };

// part[p][j] = sum over rows of part p of x[r, j]^2
template <typename T>
__global__ void __launch_bounds__(kThreads)
krylov_sumsq_kernel(int64_t n, const T* __restrict__ x, int64_t ns, int64_t chunk,
                    double* __restrict__ part) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t rb = int64_t(blockIdx.x) * chunk, re = min(n, rb + chunk);
  double acc = 0.0;
  if (j < ns)
    for (int64_t r = rb + w; r < re; r += kWarps) {
      const double v = double(x[r * ns + j]);
      acc = fma(v, v, acc);
    }
  column_part(acc, j < ns, part + int64_t(blockIdx.x) * ns + j);
}

// r -= beta[j] q_prev[:, j] (no q_prev at step 0); part[p][j] = partial q_k[:, j]^T r[:, j]
template <typename T>
__global__ void __launch_bounds__(kThreads)
krylov_three_term_kernel(int64_t n, T* __restrict__ r, const T* __restrict__ q,
                         const T* __restrict__ q_prev, const double* __restrict__ beta,
                         int64_t ns, int64_t chunk, double* __restrict__ part) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t rb = int64_t(blockIdx.x) * chunk, re = min(n, rb + chunk);
  double acc = 0.0;
  if (j < ns) {
    const double b = q_prev ? beta[j] : 0.0;
    for (int64_t row = rb + w; row < re; row += kWarps) {
      const int64_t e = row * ns + j;
      T rv = r[e];
      if (q_prev) {
        rv = T(double(rv) - b * double(q_prev[e]));
        r[e] = rv;
      }
      acc = fma(double(q[e]), double(rv), acc);
    }
  }
  column_part(acc, j < ns, part + int64_t(blockIdx.x) * ns + j);
}

// r -= alpha[j] q_k[:, j]; with `norm`, part[p][j] = partial ||r[:, j]||^2
template <typename T>
__global__ void __launch_bounds__(kThreads)
krylov_axpy_kernel(int64_t n, T* __restrict__ r, const T* __restrict__ q,
                   const double* __restrict__ alpha, int64_t ns, int64_t chunk, bool norm,
                   double* __restrict__ part) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t rb = int64_t(blockIdx.x) * chunk, re = min(n, rb + chunk);
  double acc = 0.0;
  if (j < ns) {
    const double a = alpha[j];
    for (int64_t row = rb + w; row < re; row += kWarps) {
      const int64_t e = row * ns + j;
      const T rv = T(double(r[e]) - a * double(q[e]));
      r[e] = rv;
      acc = fma(double(rv), double(rv), acc);
    }
  }
  if (norm) column_part(acc, j < ns, part + int64_t(blockIdx.x) * ns + j);
}

// Per-column Gram: part[p][i][j] = partial sum_r V[i, r, j] b[r, j] for i < kb.  CTA z takes the
// basis vectors [8z, 8z + 8).
template <typename T>
__global__ void __launch_bounds__(kThreads)
krylov_cgs_gram_kernel(int64_t n, const T* __restrict__ V, int64_t kb, const T* __restrict__ b,
                       int64_t ns, int64_t chunk, double* __restrict__ part) {
  __shared__ double sums[kWarps][kGramTile][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t i0 = int64_t(blockIdx.z) * kGramTile;
  const int64_t rb = int64_t(blockIdx.x) * chunk, re = min(n, rb + chunk);
  const int64_t plane = n * ns;
  double acc[kGramTile];
#pragma unroll
  for (int t = 0; t < kGramTile; ++t) acc[t] = 0.0;
  if (j < ns) {
    const T* vp = V + i0 * plane;
    for (int64_t row = rb + w; row < re; row += kWarps) {
      const int64_t e = row * ns + j;
      const double bv = double(b[e]);
#pragma unroll
      for (int t = 0; t < kGramTile; ++t)
        if (i0 + t < kb) acc[t] = fma(double(vp[t * plane + e]), bv, acc[t]);
    }
  }
#pragma unroll
  for (int t = 0; t < kGramTile; ++t) sums[w][t][lane] = acc[t];
  __syncthreads();
  if (w == 0 && j < ns) {
    const int64_t p = blockIdx.x;
    for (int t = 0; t < kGramTile && i0 + t < kb; ++t) {
      double s = 0.0;
      for (int q = 0; q < kWarps; ++q) s += sums[q][t][lane];
      part[(p * kb + i0 + t) * ns + j] = s;
    }
  }
}

// r[:, j] -= sum_i V[i, :, j] h[i, j] (classical Gram-Schmidt, i in order);
// part[p][j] = partial ||r[:, j]||^2 of the result
template <typename T>
__global__ void __launch_bounds__(kThreads)
krylov_cgs_update_kernel(int64_t n, const T* __restrict__ V, int64_t kb,
                         const double* __restrict__ h, T* __restrict__ r, int64_t ns,
                         int64_t chunk, double* __restrict__ part) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t rb = int64_t(blockIdx.x) * chunk, re = min(n, rb + chunk);
  const int64_t plane = n * ns;
  double acc = 0.0;
  if (j < ns)
    for (int64_t row = rb + w; row < re; row += kWarps) {
      const int64_t e = row * ns + j;
      double s = 0.0;
      for (int64_t i = 0; i < kb; ++i) s = fma(double(V[i * plane + e]), __ldg(h + i * ns + j), s);
      const T rv = T(double(r[e]) - s);
      r[e] = rv;
      acc = fma(double(rv), double(rv), acc);
    }
  column_part(acc, j < ns, part + int64_t(blockIdx.x) * ns + j);
}

// max_r sum_e |A[r, e]|: the infinity norm, a bound of the spectral radius of a symmetric A.
// Non-negative doubles order like their bit patterns, so an integer atomicMax is exact.
template <typename T>
__global__ void krylov_norm_bound_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                         const T* __restrict__ data,
                                         unsigned long long* __restrict__ out) {
  double best = 0.0;
  for (int64_t row = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; row < n;
       row += int64_t(gridDim.x) * blockDim.x) {
    double s = 0.0;
    for (int32_t e = indptr[row]; e < indptr[row + 1]; ++e) s += fabs(double(data[e]));
    best = fmax(best, s);
  }
  for (int off = 16; off > 0; off >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, off));
  if ((threadIdx.x & 31) == 0) atomicMax(out, (unsigned long long)__double_as_longlong(best));
}

// q_0 = x / ||x||: beta[j] = ||x[:, j]||, a zero column gets m = 0 and stays zero
__global__ void krylov_start_kernel(int64_t ns, const double* __restrict__ ss,
                                    double* __restrict__ beta0, int32_t* __restrict__ m,
                                    double* __restrict__ den, double* __restrict__ scale) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= ns) return;
  const double nrm = sqrt(ss[j]);
  beta0[j] = nrm;
  den[j] = nrm;
  m[j] = nrm > 0.0 ? 1 : 0;
  scale[j] = 0.0;
}

// End of step k: beta_{k+1} = ||r||.  A column that is still growing (m = k + 1) takes
// q_{k+1} = r / beta_{k+1} unless beta_{k+1} <= tol * max(largest |alpha|, |beta| so far,
// ||A||_inf); then it freezes at m = k + 1, its beta_{k+1} is stored as 0 and q_{k+1} as zeros.
__global__ void krylov_step_kernel(int64_t ns, int k, double tol,
                                   const double* __restrict__ anorm,
                                   const double* __restrict__ alpha, const double* __restrict__ ss,
                                   double* __restrict__ beta_next, int32_t* __restrict__ m,
                                   double* __restrict__ den, double* __restrict__ scale) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= ns) return;
  const double sc = fmax(scale[j], fabs(alpha[j]));
  const double b = sqrt(ss[j]);
  const bool grow = m[j] == k + 1 && b > tol * fmax(sc, *anorm);
  beta_next[j] = grow ? b : 0.0;
  den[j] = grow ? b : 0.0;
  scale[j] = grow ? fmax(sc, b) : sc;
  if (grow) m[j] = k + 2;
}

// dst[r, j] = src[r, j] / den[j], or 0 where den[j] == 0 (src may be dst)
template <typename T>
__global__ void krylov_scale_kernel(int64_t count, int64_t ns, const T* src,
                                    const double* __restrict__ den, T* dst) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < count;
       e += int64_t(gridDim.x) * blockDim.x) {
    const double d = den[e % ns];
    dst[e] = d > 0.0 ? T(double(src[e]) / d) : T(0);
  }
}

// Y[f, r, j] = sum_i V[i, r, j] W[f, i, j] for the filters [16z, 16z + 16): one pass over V
// for up to 16 filters.  Y's rows have stride ldy.
template <typename T>
__global__ void __launch_bounds__(kThreads)
krylov_combine_kernel(int64_t n, const T* __restrict__ V, int64_t kb, const double* __restrict__ W,
                      int64_t nf, int64_t ns, T* __restrict__ Y, int64_t ldy) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t row = int64_t(blockIdx.x) * kWarps + w;
  const int64_t f0 = int64_t(blockIdx.z) * kFilterTile;
  if (row >= n || j >= ns) return;
  const int64_t plane = n * ns, e = row * ns + j;
  double acc[kFilterTile];
#pragma unroll
  for (int t = 0; t < kFilterTile; ++t) acc[t] = 0.0;
  for (int64_t i = 0; i < kb; ++i) {
    const double v = double(V[i * plane + e]);
#pragma unroll
    for (int t = 0; t < kFilterTile; ++t)
      if (f0 + t < nf) acc[t] = fma(v, __ldg(W + ((f0 + t) * kb + i) * ns + j), acc[t]);
  }
#pragma unroll
  for (int t = 0; t < kFilterTile; ++t)
    if (f0 + t < nf) Y[((f0 + t) * n + row) * ldy + j] = T(acc[t]);
}

template <typename T>
int krylov_basis(int64_t n, int64_t ncols, const int32_t* indptr, const int32_t* indices,
                 const T* data, const T* x, int64_t ns, int order, T* V, double* alpha,
                 double* beta, double* vs, int32_t* m, cudaStream_t st) {
  GSP_REQUIRE(n >= 1 && ns >= 1 && order >= 1, "bad sizes");
  // the SpMM reads q_k at A's column indices: a non-square A would read outside the basis
  GSP_REQUIRE(ncols == n, "the matrix must be square");
  GSP_REQUIRE(ns <= (1 << 20), "nsig out of range");
  const int64_t cg = ceil_div(ns, 32);
  GSP_REQUIRE(ceil_div(order, kGramTile) < 65536, "order too large");
  const Parts P = row_parts(n);
  const int64_t plane = n * ns;
  // scratch: partials (P.used x order x ns), h (order x ns), ss, den, scale (ns), ||A||_inf
  const int64_t n_part = P.used * order * ns, n_h = int64_t(order) * ns;
  Scratch<double> scratch(st);
  GSP_CUDA(scratch.alloc(n_part + n_h + 3 * ns + 1));
  double *part = scratch.get(), *h = part + n_part, *ss = h + n_h, *den = ss + ns;
  double *scale = den + ns, *anorm = scale + ns;
  const dim3 red((unsigned)P.used, (unsigned)cg);
  const double tol = kBreakdown * Eps<T>::value;
  GSP_CUDA(cudaMemsetAsync(anorm, 0, sizeof(double), st));
  krylov_norm_bound_kernel<T><<<grid_for(n), kThreads, 0, st>>>(
      n, indptr, data, reinterpret_cast<unsigned long long*>(anorm));
  GSP_LAUNCH_CHECK("krylov_norm_bound");
  krylov_sumsq_kernel<T><<<red, kThreads, 0, st>>>(n, x, ns, P.chunk, part);
  GSP_LAUNCH_CHECK("krylov_sumsq");
  int rc = sum_parts(part, P.used, ns, ss, st);
  if (rc != GSP_OK) return rc;
  krylov_start_kernel<<<grid_for(ns), kThreads, 0, st>>>(ns, ss, beta, m, den, scale);
  GSP_LAUNCH_CHECK("krylov_start");
  krylov_scale_kernel<T><<<grid_for(plane), kThreads, 0, st>>>(plane, ns, x, den, V);
  GSP_LAUNCH_CHECK("krylov_scale");
  for (int k = 0; k < order; ++k) {
    const T* q = V + k * plane;
    T* r = V + (k + 1) * plane;
    if ((rc = spmm(n, indptr, indices, data, q, ns, r, st)) != GSP_OK) return rc;
    krylov_three_term_kernel<T><<<red, kThreads, 0, st>>>(
        n, r, q, k ? q - plane : nullptr, beta + int64_t(k) * ns, ns, P.chunk, part);
    GSP_LAUNCH_CHECK("krylov_three_term");
    if ((rc = sum_parts(part, P.used, ns, alpha + int64_t(k) * ns, st)) != GSP_OK) return rc;
    if (k == order - 1) break;             // beta_order and q_order are not part of the result
    krylov_axpy_kernel<T><<<red, kThreads, 0, st>>>(n, r, q, alpha + int64_t(k) * ns, ns,
                                                    P.chunk, k == 0, part);
    GSP_LAUNCH_CHECK("krylov_axpy");
    if (k > 0) {                           // full reorthogonalisation, as approximations.py:335
      const int64_t kb = k + 1;
      krylov_cgs_gram_kernel<T><<<dim3((unsigned)P.used, (unsigned)cg,
                                       (unsigned)ceil_div(kb, kGramTile)),
                                  kThreads, 0, st>>>(n, V, kb, r, ns, P.chunk, part);
      GSP_LAUNCH_CHECK("krylov_cgs_gram");
      if ((rc = sum_parts(part, P.used, kb * ns, h, st)) != GSP_OK) return rc;
      krylov_cgs_update_kernel<T><<<red, kThreads, 0, st>>>(n, V, kb, h, r, ns, P.chunk, part);
      GSP_LAUNCH_CHECK("krylov_cgs_update");
    }
    if ((rc = sum_parts(part, P.used, ns, ss, st)) != GSP_OK) return rc;
    krylov_step_kernel<<<grid_for(ns), kThreads, 0, st>>>(
        ns, k, tol, anorm, alpha + int64_t(k) * ns, ss, beta + int64_t(k + 1) * ns, m, den, scale);
    GSP_LAUNCH_CHECK("krylov_step");
    krylov_scale_kernel<T><<<grid_for(plane), kThreads, 0, st>>>(plane, ns, r, den, r);
    GSP_LAUNCH_CHECK("krylov_scale");
  }
  // V^T s, computed explicitly as the reference does (approximations.py:274)
  krylov_cgs_gram_kernel<T><<<dim3((unsigned)P.used, (unsigned)cg,
                                   (unsigned)ceil_div(order, kGramTile)),
                              kThreads, 0, st>>>(n, V, order, x, ns, P.chunk, part);
  GSP_LAUNCH_CHECK("krylov_cgs_gram");
  return sum_parts(part, P.used, int64_t(order) * ns, vs, st);
}

template <typename T>
int krylov_combine(int64_t n, const T* V, int64_t kb, const double* W, int64_t nf, int64_t ns,
                   T* Y, int64_t ldy, cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && kb >= 1 && nf >= 1 && ns >= 1 && ldy >= ns, "bad sizes");
  if (n == 0) return GSP_OK;
  const int64_t rows = ceil_div(n, kWarps), cg = ceil_div(ns, 32), ft = ceil_div(nf, kFilterTile);
  GSP_REQUIRE(rows < (int64_t(1) << 31) && cg < 65536 && ft < 65536, "block too large");
  krylov_combine_kernel<T><<<dim3((unsigned)rows, (unsigned)cg, (unsigned)ft), kThreads, 0, st>>>(
      n, V, kb, W, nf, ns, Y, ldy);
  GSP_LAUNCH_CHECK("krylov_combine");
  return GSP_OK;
}

}  // namespace
}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {

#define GSP_KRYLOV_API(SUF, T)                                                                     \
  int gsp_krylov_basis_##SUF(int64_t n, int64_t ncols, const int32_t* indptr,                     \
                             const int32_t* indices, const T* data, const T* x, int64_t nsig,     \
                             int order, T* V, double* alpha, double* beta, double* vs, int32_t* m, void* stream) {  \
    return gsp::krylov_basis<T>(n, ncols, indptr, indices, data, x, nsig, order, V, alpha, beta,  \
                                vs, m, gsp::as_stream(stream));                                    \
  }                                                                                                \
  int gsp_krylov_combine_##SUF(int64_t n, const T* V, int64_t k, const double* W, int64_t nf,     \
                               int64_t nsig, T* Y, int64_t ldy, void* stream) {                    \
    return gsp::krylov_combine<T>(n, V, k, W, nf, nsig, Y, ldy, gsp::as_stream(stream));           \
  }

GSP_KRYLOV_API(f32, float)
GSP_KRYLOV_API(f64, double)

}  // extern "C"
