// Graph multiresolution (pygsp/reduction.py): Kron reduction by independent Schur blocks,
// effective resistances of the stored edges, and the Spielman-Srivastava edge sampler.
//
// Replaces, for pygsp/reduction.py:
//   * linalg.spsolve(L_comp, L_out_in) and the product with L_in_out of kron_reduction
//     (:358), one sparse direct solve over all removed vertices  -> gsp_schur_small_f64 (one CTA
//     per small component of the removed vertices), gsp_schur_gather_f64 (dense blocks of a
//     large component for the caller's float64 Cholesky)
//   * resistance_distances[start_nodes, end_nodes] of graph_sparsify (:84, :101)
//                                                                  -> gsp_edge_resistance_f64
//   * stats.rv_discrete(...).rvs(size=q) and the removed stats.itemfreq (:104-115)
//                                                                  -> gsp_sparsify_sample
//
// Schur blocks.  Write S for one connected component of the removed vertices (connected through
// the stored off-diagonal entries of M) and B for its kept neighbours.  Then
//   M_red - M_io M_comp^-1 M_oi = M_red - sum_S M_BS M_SS^-1 M_SB
// and, with M_SS = C C^T (Cholesky) and Y = C^-1 M_SB (s x b), the block of S is -Y^T Y: a dense
// b x b block written as b^2 COO triplets (row-major over B x B, B in increasing kept index).
// Entry (i, j) is the fma chain sum_k Y[k][i] Y[k][j] in k order, which is the same chain as
// entry (j, i): every block is exactly symmetric.
//
// Small component kernel: one CTA per component, M_SS and M_SB gathered into shared memory
// (zero-filled, then one thread per local row scatters its CSR row), a right-looking Cholesky
// in place (one column per round, three barriers per column), the forward substitution with
// one thread per column of M_SB, and the b^2 outputs with one thread per entry.  Byte/flop
// model per component, s = |S|, b = |B|, nnz_S = stored entries of S's rows:
//   HBM reads  12 nnz_S bytes (index + value) + 4 (s + b)       (the CSR rows, slots, B)
//   HBM writes 16 b^2 bytes                                      (int32 row, int32 col, f64)
//   flops      s^3 / 3 + s^2 b + s b^2                           (Cholesky, solve, Y^T Y)
// For the k-NN graphs of DESIGN section 4.11 the writes dominate: b is several times s.
//
// A non-positive pivot (M_SS not positive definite) sets *status to 1 and continues with a
// unit pivot so that nothing non-finite is written; the caller raises.
//
// Sampler.  The weights are integers k_e (the caller quantises w_e R_e); an inclusive scan in
// uint64 gives the cumulative table, exact and independent of the scan's partition.  Draw d
// belongs to chunk d / kDrawsPerChunk; each chunk owns Philox subsequence `chunk` of `seed`
// (curand_kernel.h), so a draw's value depends on (seed, d) only, whatever the launch shape.
// A 64-bit uniform r picks u = floor(r T / 2^64) in [0, T) and the edge whose interval of the
// cumulative table holds u.  Counts are integer atomics: the same seed gives the same counts.
#include <cub/cub.cuh>
#include <curand_kernel.h>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {
namespace {

constexpr int kSchurThreads = 256;
constexpr int64_t kDrawsPerChunk = 128;   // one thread per chunk: q / 128 threads
constexpr int kSampleThreads = 128;

// position of `key` in the sorted list b[0..nb), -1 if absent
__device__ __forceinline__ int find_sorted(const int32_t* b, int nb, int key) {
  int lo = 0, hi = nb;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (b[mid] < key) lo = mid + 1; else hi = mid;
  }
  return (lo < nb && b[lo] == key) ? lo : -1;
}

// slot[v] >= 0: v is removed, slot = its position in its component; slot[v] < 0: v is kept with
// index -slot - 1.  Scatters M_SS (s x s) and M_SB (s x b) of the component whose vertices are
// cvert[0..s) into A (lda) and Bm (ldb), both zero on entry.
__device__ __forceinline__ void gather_rows(int row0, int row_step, int s, int nb,
                                            const int32_t* __restrict__ indptr,
                                            const int32_t* __restrict__ indices,
                                            const double* __restrict__ data,
                                            const int32_t* __restrict__ slot,
                                            const int32_t* __restrict__ cvert,
                                            const int32_t* bids, double* A, int64_t lda,
                                            double* Bm, int64_t ldb) {
  for (int i = row0; i < s; i += row_step) {
    const int v = __ldg(cvert + i);
    const int end = __ldg(indptr + v + 1);
    for (int k = __ldg(indptr + v); k < end; ++k) {
      const int u = __ldg(indices + k);
      const int sl = __ldg(slot + u);
      const double w = __ldg(data + k);
      if (sl >= 0) {
        A[int64_t(i) * lda + sl] = w;
      } else {
        const int j = find_sorted(bids, nb, -sl - 1);
        if (j >= 0) Bm[int64_t(i) * ldb + j] = w;
      }
    }
  }
}

__global__ void __launch_bounds__(kSchurThreads)
schur_small_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                   const double* __restrict__ data, const int32_t* __restrict__ slot,
                   const int32_t* __restrict__ cvert, const int32_t* __restrict__ cptr,
                   const int32_t* __restrict__ bptr, const int32_t* __restrict__ bidx,
                   const int32_t* __restrict__ comps, const int64_t* __restrict__ out_off,
                   int32_t* rows, int32_t* cols, double* vals, int32_t* status) {
  extern __shared__ double smem[];
  const int c = __ldg(comps + blockIdx.x);
  const int c0 = __ldg(cptr + c), s = __ldg(cptr + c + 1) - c0;
  const int b0 = __ldg(bptr + c), nb = __ldg(bptr + c + 1) - b0;
  double* C = smem;                       // s x s, lower Cholesky factor in place
  double* rinv = C + s * s;               // s, reciprocals of the pivots
  double* Y = rinv + s;                   // s x nb, M_SB then C^-1 M_SB
  int32_t* bids = reinterpret_cast<int32_t*>(Y + s * nb);
  const int tid = threadIdx.x;

  for (int e = tid; e < s * s + s + s * nb; e += blockDim.x) smem[e] = 0.0;
  for (int e = tid; e < nb; e += blockDim.x) bids[e] = __ldg(bidx + b0 + e);
  __syncthreads();
  gather_rows(tid, blockDim.x, s, nb, indptr, indices, data, slot, cvert + c0, bids, C, s, Y, nb);
  __syncthreads();

  // right-looking Cholesky: C[i][k] for k <= i
  for (int j = 0; j < s; ++j) {
    if (tid == 0) {
      double d = C[j * s + j];
      if (!(d > 0.0)) {
        *status = 1;
        d = 1.0;
      }
      d = sqrt(d);
      C[j * s + j] = d;
      rinv[j] = __drcp_rn(d);     // a multiply by the reciprocal: no division subroutine
    }
    __syncthreads();
    const double r = rinv[j];
    for (int i = j + 1 + tid; i < s; i += blockDim.x) C[i * s + j] *= r;
    __syncthreads();
    const int m = s - j - 1;
    for (int e = tid; e < m * m; e += blockDim.x) {
      const int i = j + 1 + e / m, k = j + 1 + e % m;
      if (k <= i) C[i * s + k] = fma(-C[i * s + j], C[k * s + j], C[i * s + k]);
    }
    __syncthreads();
  }

  // Y := C^-1 M_SB, one thread per column
  for (int t = tid; t < nb; t += blockDim.x) {
    for (int i = 0; i < s; ++i) {
      double acc = Y[i * nb + t];
      for (int k = 0; k < i; ++k) acc = fma(-C[i * s + k], Y[k * nb + t], acc);
      Y[i * nb + t] = acc * rinv[i];
    }
  }
  __syncthreads();

  // -Y^T Y, row-major over B x B
  const int64_t base = __ldg(out_off + c);
  for (int e = tid; e < nb * nb; e += blockDim.x) {
    const int i = e / nb, j = e % nb;
    double acc = 0.0;
    for (int k = 0; k < s; ++k) acc = fma(Y[k * nb + i], Y[k * nb + j], acc);
    rows[base + e] = bids[i];
    cols[base + e] = bids[j];
    vals[base + e] = -acc;
  }
}

__global__ void schur_gather_kernel(const int32_t* __restrict__ indptr,
                                    const int32_t* __restrict__ indices,
                                    const double* __restrict__ data,
                                    const int32_t* __restrict__ slot,
                                    const int32_t* __restrict__ cvert, int s,
                                    const int32_t* __restrict__ bidx, int nb, double* A,
                                    double* Bm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  gather_rows(i, gridDim.x * blockDim.x, s, nb, indptr, indices, data, slot, cvert, bidx, A, s,
              Bm, nb);
}

__global__ void edge_resistance_kernel(int64_t ne, const int32_t* __restrict__ erow,
                                       const int32_t* __restrict__ ecol,
                                       const double* __restrict__ ainv, int64_t lda,
                                       double* R) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= ne) return;
  const int64_t u = __ldg(erow + e), v = __ldg(ecol + e);
  const double uu = __ldg(ainv + u * lda + u), vv = __ldg(ainv + v * lda + v);
  const double uv = __ldg(ainv + u * lda + v), vu = __ldg(ainv + v * lda + u);
  R[e] = (uu + vv) - (uv + vu);
}

__global__ void __launch_bounds__(kSampleThreads)
sample_kernel(int64_t ne, const unsigned long long* __restrict__ cum, int64_t q, uint64_t seed,
              unsigned long long* counts) {
  const int64_t chunk = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t d0 = chunk * kDrawsPerChunk;
  if (d0 >= q) return;
  const int64_t d1 = d0 + kDrawsPerChunk < q ? d0 + kDrawsPerChunk : q;
  const unsigned long long total = __ldg(cum + ne - 1);
  curandStatePhilox4_32_10_t state;
  curand_init(seed, (unsigned long long)chunk, 0ull, &state);
  for (int64_t d = d0; d < d1; d += 2) {
    const uint4 r = curand4(&state);
    const unsigned long long r0 = (uint64_t(r.x) << 32) | r.y, r1 = (uint64_t(r.z) << 32) | r.w;
    for (int h = 0; h < 2 && d + h < d1; ++h) {
      const unsigned long long u = __umul64hi(h ? r1 : r0, total);
      // first e with cum[e] > u
      int64_t lo = 0, hi = ne - 1;
      while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(cum + mid) > u) hi = mid; else lo = mid + 1;
      }
      atomicAdd(counts + lo, 1ull);
    }
  }
}

}  // namespace

int schur_small(const int32_t* indptr, const int32_t* indices, const double* data,
                const int32_t* slot, const int32_t* cvert, const int32_t* cptr,
                const int32_t* bptr, const int32_t* bidx, int64_t n_small, const int32_t* comps,
                int smem_bytes, const int64_t* out_off, int32_t* rows, int32_t* cols,
                double* vals, int32_t* status, cudaStream_t st) {
  GSP_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
  if (n_small == 0) return GSP_OK;
  GSP_CUDA(cudaFuncSetAttribute(schur_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                smem_bytes));
  schur_small_kernel<<<(unsigned)n_small, kSchurThreads, smem_bytes, st>>>(
      indptr, indices, data, slot, cvert, cptr, bptr, bidx, comps, out_off, rows, cols, vals,
      status);
  GSP_LAUNCH_CHECK("schur_small");
  return GSP_OK;
}

int schur_gather(const int32_t* indptr, const int32_t* indices, const double* data,
                 const int32_t* slot, const int32_t* cvert, int64_t s, const int32_t* bidx,
                 int64_t nb, double* A, double* Bm, cudaStream_t st) {
  GSP_CUDA(cudaMemsetAsync(A, 0, sizeof(double) * s * s, st));
  if (nb) GSP_CUDA(cudaMemsetAsync(Bm, 0, sizeof(double) * s * nb, st));
  if (s == 0) return GSP_OK;
  schur_gather_kernel<<<(int)ceil_div(s, 128), 128, 0, st>>>(indptr, indices, data, slot, cvert,
                                                             (int)s, bidx, (int)nb, A, Bm);
  GSP_LAUNCH_CHECK("schur_gather");
  return GSP_OK;
}

int edge_resistance(int64_t ne, const int32_t* erow, const int32_t* ecol, const double* ainv,
                    int64_t lda, double* R, cudaStream_t st) {
  if (ne == 0) return GSP_OK;
  edge_resistance_kernel<<<(int)ceil_div(ne, 256), 256, 0, st>>>(ne, erow, ecol, ainv, lda, R);
  GSP_LAUNCH_CHECK("edge_resistance");
  return GSP_OK;
}

int sparsify_sample(int64_t ne, const uint64_t* weights, int64_t q, uint64_t seed,
                    int64_t* counts, cudaStream_t st) {
  GSP_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * ne, st));
  if (ne == 0 || q == 0) return GSP_OK;
  Scratch<unsigned long long> cum(st);
  GSP_CUDA(cum.alloc(ne));
  const unsigned long long* w = reinterpret_cast<const unsigned long long*>(weights);
  const int rc = cub_temp("cub::DeviceScan::InclusiveSum", st, [&](void* tmp, size_t& bytes) {
    return cub::DeviceScan::InclusiveSum(tmp, bytes, w, cum.get(), (int)ne, st);
  });
  if (rc != GSP_OK) return rc;
  const int64_t chunks = ceil_div(q, kDrawsPerChunk);
  sample_kernel<<<(int)ceil_div(chunks, kSampleThreads), kSampleThreads, 0, st>>>(
      ne, cum.get(), q, seed, reinterpret_cast<unsigned long long*>(counts));
  GSP_LAUNCH_CHECK("sparsify_sample");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {
int gsp_schur_small_f64(const int32_t* indptr, const int32_t* indices, const double* data,
                        const int32_t* slot, const int32_t* cvert, const int32_t* cptr,
                        const int32_t* bptr, const int32_t* bidx, int64_t n_small,
                        const int32_t* comps, int smem_bytes, const int64_t* out_off,
                        int32_t* rows, int32_t* cols, double* vals, int32_t* status,
                        void* stream) {
  GSP_REQUIRE(n_small >= 0 && n_small < (int64_t(1) << 31) && status, "bad arguments");
  GSP_REQUIRE(smem_bytes >= 0 && smem_bytes <= 227 * 1024, "shared memory out of range");
  return gsp::schur_small(indptr, indices, data, slot, cvert, cptr, bptr, bidx, n_small, comps,
                          smem_bytes, out_off, rows, cols, vals, status, gsp::as_stream(stream));
}
int gsp_schur_gather_f64(const int32_t* indptr, const int32_t* indices, const double* data,
                         const int32_t* slot, const int32_t* cvert, int64_t s,
                         const int32_t* bidx, int64_t nb, double* A, double* B, void* stream) {
  GSP_REQUIRE(s >= 0 && s < (int64_t(1) << 31) && nb >= 0 && nb < (int64_t(1) << 31),
              "bad arguments");
  return gsp::schur_gather(indptr, indices, data, slot, cvert, s, bidx, nb, A, B,
                           gsp::as_stream(stream));
}
int gsp_edge_resistance_f64(int64_t ne, const int32_t* erow, const int32_t* ecol,
                            const double* ainv, int64_t lda, double* R, void* stream) {
  GSP_REQUIRE(ne >= 0 && lda >= 0, "bad arguments");
  return gsp::edge_resistance(ne, erow, ecol, ainv, lda, R, gsp::as_stream(stream));
}
int gsp_sparsify_sample(int64_t ne, const uint64_t* weights, int64_t q, uint64_t seed,
                        int64_t* counts, void* stream) {
  GSP_REQUIRE(ne >= 0 && ne < (int64_t(1) << 31) && q >= 0, "bad arguments");
  return gsp::sparsify_sample(ne, weights, q, seed, counts, gsp::as_stream(stream));
}
}
