// Filter banks wider than kMaxScales (16): analysis through a stored Chebyshev basis, synthesis
// through per-order sources and one Clenshaw recurrence.
//
// Analysis (approximations.py:58-114 for a wide bank).  gsp_cheby_op_* applies the fused step to
// the first 16 filters and then reads and writes every other accumulator block once per order
// (cheby_axpy_scales): about (m - 1)(2 Nf + 4) passes over the (n, nsig) block.  Here the m - 1
// recurrence steps run with no accumulator and write T_k x into slot k of a basis buffer
// (m, n, nsig) -- each step through run_step, so the tiled kernel applies as for any step -- and
// one combine pass forms every r_i = sum_k c_ik T_k x: about 4 (m - 1) + m + Nf passes.
//
// Synthesis (filter.py:313-322 for more than 16 features).  The mix pass forms the per-order
// sources u_k = sum_f c'_fk s_f (c'_f0 = c_f0 / 2) in one read of the Nf source blocks, and ONE
// Clenshaw recurrence with a per-order source, b_k = u_k + 2 Lt b_{k+1} - b_{k+2}, is the
// add_source step with a single source block whose pointer moves with k: m - 1 SpMMs in all,
// instead of Nf (m - 1) for the reference's Nf forward recurrences.
#include <algorithm>
#include "step.cuh"

namespace gsp {

constexpr int kCombineThreads = 128;   // most threads per CTA of the combine kernel
constexpr int kMixThreads = 256;
constexpr int kMixFilters = 32;        // coefficient rows staged in shared memory at a time

// r_i = sum_k c_ik T_k x over the elements of a (n, nsig) block, VEC consecutive elements per
// thread, for the orders k0 .. k1 - 1 of one chunk.  The CTA stages the basis values of its
// elements for these orders in shared memory once (each thread reads back only what it staged, so
// no barrier is needed) and loops over all nscales filters; the coefficient rows are read from L2
// as doubles.  The chain is the fused step's, with the coefficients cast to T as StepCoef casts
// them:
//   r = fma(c_i1, T_1, T(c_i0 / 2) T_0), then r = fma(c_ik, T_k, r) for k = 2 .. m-1
// so the result is the bits of gsp_cheby_op_* on the same block.  A chunk past the first
// (k0 > 0) continues the chain from the r the previous chunk stored: r is a T value, so storing
// and reloading it changes no bit.
template <typename T, int VEC>
__global__ void __launch_bounds__(kCombineThreads)
cheby_basis_combine(int64_t count, int nsig, const T* __restrict__ t0, const T* __restrict__ basis,
                    int m, int k0, int k1, const double* __restrict__ coeffs, int nscales,
                    T* __restrict__ r, int64_t r_stride, int64_t ldr) {
  extern __shared__ __align__(16) unsigned char combine_smem[];
  Vec<T, VEC>* tile = reinterpret_cast<Vec<T, VEC>*>(combine_smem);   // (k1 - k0, blockDim.x)
  const int tpb = blockDim.x;
  const int64_t e = (int64_t(blockIdx.x) * tpb + threadIdx.x) * VEC;
  if (e >= count) return;
  Vec<T, VEC>* mine = tile + threadIdx.x;                  // slot k - k0 holds T_k
  for (int k = k0; k < k1; ++k)
    mine[(k - k0) * tpb] = load_vec_stream<T, VEC>(k == 0 ? t0 + e : basis + int64_t(k) * count + e);
  const int64_t row = e / nsig;
  T* out = r + row * ldr + (e - row * nsig);
  for (int i = 0; i < nscales; ++i) {
    const double* ci = coeffs + int64_t(i) * m;
    T* oi = out + int64_t(i) * r_stride;
    Vec<T, VEC> acc;
    if (k0 == 0) {
      const T h0 = T(0.5 * __ldg(ci));
      const T c1 = T(__ldg(ci + 1));
      const Vec<T, VEC> x0 = mine[0], x1 = mine[tpb];
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc.v[v] = fma(c1, x1.v[v], h0 * x0.v[v]);
    } else {
      acc = load_vec_stream<T, VEC>(oi);
    }
#pragma unroll 4
    for (int k = max(k0, 2); k < k1; ++k) {
      const T ck = T(__ldg(ci + k));
      const Vec<T, VEC> xk = mine[(k - k0) * tpb];
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc.v[v] = fma(ck, xk.v[v], acc.v[v]);
    }
    store_vec_stream<T, VEC>(oi, acc);
  }
}

// u_k = sum_f c'_fk s_f for the KP orders k0 .. k0 + kn - 1 (kn <= KP), c'_f0 = c_f0 / 2: one
// thread per element, its KP accumulators in registers, the sum in increasing f.  The coefficient
// rows are staged in shared memory, cast to T, kMixFilters rows at a time.
template <typename T, int KP>
__global__ void __launch_bounds__(kMixThreads)
cheby_mix_orders(int64_t count, const T* __restrict__ src, int nsrc, const double* __restrict__ coeffs,
                 int m, int k0, int kn, T* __restrict__ u) {
  __shared__ T cs[kMixFilters][KP];
  const int64_t e = int64_t(blockIdx.x) * kMixThreads + threadIdx.x;
  const bool active = e < count;
  T acc[KP];
#pragma unroll
  for (int k = 0; k < KP; ++k) acc[k] = T(0);
  for (int f0 = 0; f0 < nsrc; f0 += kMixFilters) {
    const int fn = min(kMixFilters, nsrc - f0);
    __syncthreads();
    for (int t = threadIdx.x; t < kMixFilters * KP; t += kMixThreads) {
      const int f = t / KP, k = t - (t / KP) * KP;
      double c = 0.0;
      if (f < fn && k < kn) {
        c = __ldg(coeffs + int64_t(f0 + f) * m + k0 + k);
        if (k0 + k == 0) c = 0.5 * c;
      }
      cs[f][k] = T(c);
    }
    __syncthreads();
    if (!active) continue;
#pragma unroll 4
    for (int f = 0; f < fn; ++f) {
      const T s = __ldcs(src + int64_t(f0 + f) * count + e);
#pragma unroll
      for (int k = 0; k < KP; ++k) acc[k] = fma(cs[f][k], s, acc[k]);
    }
  }
  if (!active) return;
#pragma unroll
  for (int k = 0; k < KP; ++k)
    if (k < kn) __stcs(u + int64_t(k0 + k) * count + e, acc[k]);
}

// The combine in order chunks.  The thread count halves from 128 to 32 while the m staged values of
// a thread do not fit in the shared-memory opt-in (m <= 113, 227, 454 at 16 B per value, the
// vectorised case in both types); past that the orders are split into chunks of as many as fit
// at 32 threads, each launch continuing the chains of the one before.
template <typename T, int VEC>
static int launch_combine(int64_t count, int nsig, const T* t0, const T* basis, int m,
                          const double* coeffs, int nscales, T* r, int64_t r_stride, int64_t ldr,
                          cudaStream_t st) {
  int dev = 0, optin = 0;
  GSP_CUDA(cudaGetDevice(&dev));
  GSP_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const int64_t per_order = int64_t(VEC) * sizeof(T);      // bytes per thread and order
  int tpb = kCombineThreads;
  while (tpb > 32 && per_order * m * tpb > optin) tpb /= 2;
  const int chunk = int(std::min<int64_t>(m, optin / (per_order * tpb)));
  GSP_REQUIRE(chunk >= 2, "basis combine: no shared memory for two orders");
  const size_t smem = size_t(per_order) * chunk * tpb;
  GSP_CUDA(cudaFuncSetAttribute(cheby_basis_combine<T, VEC>,
                                cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t blocks = ceil_div(count, int64_t(tpb) * VEC);
  GSP_REQUIRE(blocks < (int64_t(1) << 31), "block too large for one combine launch");
  for (int k0 = 0; k0 < m; k0 += chunk) {
    const int k1 = std::min(m, k0 + chunk);
    cheby_basis_combine<T, VEC><<<(unsigned)blocks, tpb, size_t(per_order) * (k1 - k0) * tpb, st>>>(
        count, nsig, t0, basis, m, k0, k1, coeffs, nscales, r, r_stride, ldr);
    GSP_LAUNCH_CHECK("cheby_basis_combine");
  }
  return GSP_OK;
}

template <typename T> struct BankVec;
template <> struct BankVec<float> { static constexpr int value = 4; };
template <> struct BankVec<double> { static constexpr int value = 2; };

// Forward recurrence into the basis, then the combine pass (gsp_cheby_op_basis_*).
template <typename T>
int cheby_op_basis(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                   const T* vals, double lmax, const double* coeffs, int nscales, int m, const T* x,
                   int nsig, T* basis, T* r, int64_t ldr, const gsp_tile_plan* plan, cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && nsig >= 1 && nscales >= 1 && ldr >= nsig, "bad sizes");
  GSP_REQUIRE(m >= 2, "The coefficients have an invalid shape");   // approximations.py:83-84
  GSP_REQUIRE(lmax > 0 && lmax == lmax, "lmax must be positive");
  GSP_REQUIRE(coeffs && basis && r && x, "null block");
  if (n == 0) return GSP_OK;
  const int64_t count = n * int64_t(nsig);
  Step<T> s{nnz, indptr, indices, vals};
  s.r_rows = n;
  s.nsig = nsig;
  for (int k = 1; k < m; ++k) {
    // T_k = (4/lmax) L T_{k-1} - 2 T_{k-1} - T_{k-2} (k = 1: (2/lmax) L x - x) into slot k
    forward_coefs(s, k, m, 0, lmax, coeffs, nullptr, nullptr);
    s.x_cur = k == 1 ? x : basis + int64_t(k - 1) * count;
    s.x_old = k == 1 ? nullptr : (k == 2 ? x : basis + int64_t(k - 2) * count);
    s.x_new = basis + int64_t(k) * count;
    int rc = run_step<T>(s, 0, n, plan, nullptr, st);
    if (rc != GSP_OK) return rc;
  }
  constexpr int V = BankVec<T>::value;
  const bool vec_ok = nsig % V == 0 && ldr % V == 0 && aligned16(x) && aligned16(basis) &&
                      aligned16(r);
  const int64_t r_stride = n * ldr;
  if (vec_ok) return launch_combine<T, V>(count, nsig, x, basis, m, coeffs, nscales, r, r_stride, ldr, st);
  return launch_combine<T, 1>(count, nsig, x, basis, m, coeffs, nscales, r, r_stride, ldr, st);
}

template <typename T, int KP>
static int launch_mix(int64_t count, const T* src, int nsrc, const double* coeffs, int m, int k0,
                      int kn, T* u, cudaStream_t st) {
  const int64_t blocks = ceil_div(count, kMixThreads);
  GSP_REQUIRE(blocks < (int64_t(1) << 31), "block too large for one mix launch");
  cheby_mix_orders<T, KP><<<(unsigned)blocks, kMixThreads, 0, st>>>(count, src, nsrc, coeffs, m, k0,
                                                                    kn, u);
  GSP_LAUNCH_CHECK("cheby_mix_orders");
  return GSP_OK;
}

// Mix passes, then Clenshaw's recurrence with the per-order source (gsp_cheby_synthesis_wide_*).
template <typename T>
int cheby_synthesis_wide(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                         const T* vals, double lmax, const double* coeffs, int nsrc, int m,
                         const T* src, int nsig, T* out, T* work, const gsp_tile_plan* plan,
                         cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && nsig >= 1 && nsrc >= 1, "bad sizes");
  GSP_REQUIRE(m >= 2, "The coefficients have an invalid shape");
  GSP_REQUIRE(lmax > 0 && lmax == lmax, "lmax must be positive");
  GSP_REQUIRE(coeffs && src && out && work, "null block");
  if (n == 0) return GSP_OK;
  const int64_t count = n * int64_t(nsig);
  T* u = work;                                                  // u_0 .. u_K
  T* b[2] = {work + int64_t(m) * count, work + int64_t(m + 1) * count};
  for (int k0 = 0; k0 < m; k0 += 32) {
    const int kn = std::min(32, m - k0);
    const int rc = kn <= 8    ? launch_mix<T, 8>(count, src, nsrc, coeffs, m, k0, kn, u, st)
                   : kn <= 16 ? launch_mix<T, 16>(count, src, nsrc, coeffs, m, k0, kn, u, st)
                              : launch_mix<T, 32>(count, src, nsrc, coeffs, m, k0, kn, u, st);
    if (rc != GSP_OK) return rc;
  }
  const int K = m - 1;
  const double one = 1.0;
  Step<T> s{nnz, indptr, indices, vals};
  s.r_rows = n;
  s.nsig = nsig;
  s.first = false;
  s.nscales = 1;
  s.ck = &one;
  s.add_source = true;
  const T* b_cur = u + int64_t(K) * count;                      // b_K = u_K
  const T* b_old = nullptr;
  for (int k = K - 1; k >= 0; --k) {
    // middle: b_k = (4/lmax) L b_{k+1} - 2 b_{k+1} - b_{k+2} + u_k
    // last  : out = (2/lmax) L b_1 - b_1 - b_2 + u_0             (u_0 holds the halved c_f0)
    const bool last = k == 0;
    s.alpha = last ? 2.0 / lmax : 4.0 / lmax;
    s.beta = last ? -1.0 : -2.0;
    s.gamma = b_old ? -1.0 : 0.0;
    s.reverse = (k & 1) == 0;
    s.r = u + int64_t(k) * count;
    T* dst = last ? out : b[(K - 1 - k) & 1];                   // b_k over b_{k+2} (row-local)
    s.x_cur = b_cur;
    s.x_old = b_old ? b_old : b_cur;                            // no b_{k+2}: times gamma = 0
    s.x_new = dst;
    int rc = run_step<T>(s, 0, n, plan, nullptr, st);
    if (rc != GSP_OK) return rc;
    b_old = b_cur;
    b_cur = dst;
  }
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {

#define GSP_BANK_API(SUF, T)                                                                       \
  int gsp_cheby_op_basis_##SUF(int64_t n, int64_t nnz, const int32_t* indptr,                      \
                               const int32_t* indices, const T* data, double lmax,                 \
                               const double* coeffs, int nscales, int m, const T* x, int64_t nsig, \
                               T* basis, T* r, int64_t ldr, const gsp_tile_plan* plan_host,        \
                               void* stream) {                                                     \
    GSP_REQUIRE(nsig >= 1 && nsig <= (1 << 20), "nsig out of range");                              \
    return gsp::cheby_op_basis<T>(n, nnz, indptr, indices, data, lmax, coeffs, nscales, m, x,     \
                                  (int)nsig, basis, r, ldr, plan_host, gsp::as_stream(stream));    \
  }                                                                                                \
  int gsp_cheby_synthesis_wide_##SUF(int64_t n, int64_t nnz, const int32_t* indptr,                \
                                     const int32_t* indices, const T* data, double lmax,           \
                                     const double* coeffs, int nsrc, int m, const T* sources,      \
                                     int64_t nsig, T* out, T* work,                                \
                                     const gsp_tile_plan* plan_host, void* stream) {               \
    GSP_REQUIRE(nsig >= 1 && nsig <= (1 << 20), "nsig out of range");                              \
    return gsp::cheby_synthesis_wide<T>(n, nnz, indptr, indices, data, lmax, coeffs, nsrc, m,     \
                                        sources, (int)nsig, out, work, plan_host,                  \
                                        gsp::as_stream(stream));                                   \
  }

GSP_BANK_API(f32, float)
GSP_BANK_API(f64, double)

}  // extern "C"
