// Tall-skinny block kernels of the graph Fourier basis (pygsp_b200/graphs/fourier.py).
//
// Replaces, for pygsp/graphs/fourier.py:
//   * np.tensordot(U, s, ([0], [0]))     gft  (fourier.py:229-230)       -> gsp_block_gram_*
//   * np.tensordot(U, s_hat, ([1], [0])) igft (fourier.py:264)           -> gsp_block_combine_*
//   * the dense block algebra that ARPACK runs inside eigsh (fourier.py:175): Gram matrices,
//     basis rotations and residual norms of the partial eigensolver (Chebyshev-filtered
//     subspace iteration, whose filter is the fused recurrence step of csrc/cheby.cu).
//
// Blocks are row-major (n, k) in float or double; small matrices are double, row-major.
// Products accumulate in double, also for float blocks.  Every reduction over rows is
// two-level and ORDER-FIXED (csrc/reduce.cuh): CTA p reduces rows [p*chunk, (p+1)*chunk) in row
// order into a partial, sum_parts adds the partials in p order.  The partition depends only on
// the shapes, never on the device, so results are bit-reproducible.
//
// The products are register-tiled: a CTA of 16 x 16 threads owns a (16 MT) x (16 MT) output
// tile, thread (ty, tx) the MT x MT entries (ty + 16 p, tx + 16 q) -- strided, so a warp's
// shared-memory reads are one broadcast and one 128-byte line.  Slabs of KS rows (Gram) or KS
// inner indices (combine) are staged in shared memory as double.
#include "reduce.cuh"

namespace gsp {
namespace {

constexpr int kBlockThreads = 256;                  // 16 x 16 threads of a tiled product

template <int MT> struct Tile {
  static constexpr int T = 16 * MT;                 // output tile edge
  static constexpr int KS = MT == 8 ? 16 : 32;      // staged slab depth (32 KB of shared memory)
};

// micro tile: the widest output edge of a call selects it
inline int micro_tile(int64_t a, int64_t b) {
  const int64_t w = std::max(a, b);
  return w <= 32 ? 2 : (w <= 64 ? 4 : 8);
}

// part[p][i][j] = sum over rows r of part p of A[r, i] * B[r, j]
template <typename T, int MT>
__global__ void __launch_bounds__(kBlockThreads)
block_gram_kernel(int64_t n, const T* __restrict__ A, int64_t ka, const T* __restrict__ B,
                  int64_t kb, int64_t chunk, double* __restrict__ part) {
  constexpr int TT = Tile<MT>::T, KS = Tile<MT>::KS;
  __shared__ double sa[KS][TT];
  __shared__ double sb[KS][TT];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t p = blockIdx.x;
  const int64_t i0 = int64_t(blockIdx.y) * TT, j0 = int64_t(blockIdx.z) * TT;
  const int64_t rb = p * chunk, re = min(n, rb + chunk);
  double acc[MT][MT];
#pragma unroll
  for (int a = 0; a < MT; ++a)
#pragma unroll
    for (int b = 0; b < MT; ++b) acc[a][b] = 0.0;

  for (int64_t r0 = rb; r0 < re; r0 += KS) {
    for (int e = threadIdx.x; e < KS * TT; e += kBlockThreads) {
      const int r = e / TT, c = e % TT;
      const int64_t row = r0 + r;
      const bool in = row < re;
      sa[r][c] = (in && i0 + c < ka) ? double(A[row * ka + i0 + c]) : 0.0;
      sb[r][c] = (in && j0 + c < kb) ? double(B[row * kb + j0 + c]) : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      double va[MT], vb[MT];
#pragma unroll
      for (int a = 0; a < MT; ++a) va[a] = sa[kk][ty + 16 * a];
#pragma unroll
      for (int b = 0; b < MT; ++b) vb[b] = sb[kk][tx + 16 * b];
#pragma unroll
      for (int a = 0; a < MT; ++a)
#pragma unroll
        for (int b = 0; b < MT; ++b) acc[a][b] = fma(va[a], vb[b], acc[a][b]);
    }
    __syncthreads();
  }
  double* out = part + p * ka * kb;
#pragma unroll
  for (int a = 0; a < MT; ++a) {
    const int64_t i = i0 + ty + 16 * a;
    if (i >= ka) continue;
#pragma unroll
    for (int b = 0; b < MT; ++b) {
      const int64_t j = j0 + tx + 16 * b;
      if (j < kb) out[i * kb + j] = acc[a][b];
    }
  }
}

// Y[r, j] = sum_i A[r, i] Q[i, j]
template <typename T, int MT>
__global__ void __launch_bounds__(kBlockThreads)
block_combine_kernel(int64_t n, const T* __restrict__ A, int64_t ka, const double* __restrict__ Q,
                     int64_t kq, T* __restrict__ Y) {
  constexpr int TT = Tile<MT>::T, KS = Tile<MT>::KS;
  __shared__ double sa[TT][KS];
  __shared__ double sq[KS][TT];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t r0 = int64_t(blockIdx.x) * TT, j0 = int64_t(blockIdx.y) * TT;
  double acc[MT][MT];
#pragma unroll
  for (int a = 0; a < MT; ++a)
#pragma unroll
    for (int b = 0; b < MT; ++b) acc[a][b] = 0.0;

  for (int64_t k0 = 0; k0 < ka; k0 += KS) {
    for (int e = threadIdx.x; e < KS * TT; e += kBlockThreads) {
      const int r = e / KS, c = e % KS;             // A tile: TT rows x KS inner indices
      sa[r][c] = (r0 + r < n && k0 + c < ka) ? double(A[(r0 + r) * ka + k0 + c]) : 0.0;
      const int qi = e / TT, qj = e % TT;           // Q slab: KS inner indices x TT columns
      sq[qi][qj] = (k0 + qi < ka && j0 + qj < kq) ? Q[(k0 + qi) * kq + j0 + qj] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      double va[MT], vq[MT];
#pragma unroll
      for (int a = 0; a < MT; ++a) va[a] = sa[ty + 16 * a][kk];
#pragma unroll
      for (int b = 0; b < MT; ++b) vq[b] = sq[kk][tx + 16 * b];
#pragma unroll
      for (int a = 0; a < MT; ++a)
#pragma unroll
        for (int b = 0; b < MT; ++b) acc[a][b] = fma(va[a], vq[b], acc[a][b]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < MT; ++a) {
    const int64_t r = r0 + ty + 16 * a;
    if (r >= n) continue;
#pragma unroll
    for (int b = 0; b < MT; ++b) {
      const int64_t j = j0 + tx + 16 * b;
      if (j < kq) Y[r * kq + j] = T(acc[a][b]);
    }
  }
}

// part[p][j] = sum over rows r of part p of (LX[r, j] - theta[j] X[r, j])^2.
// Lane = column (32 per CTA column group), warp w takes rows w, w + 8, ...; the 8 warp sums
// are added in warp order (the order of column_part, csrc/reduce.cuh).
template <typename T>
__global__ void __launch_bounds__(kThreads)
block_residual_kernel(int64_t n, const T* __restrict__ X, const T* __restrict__ LX,
                      const double* __restrict__ theta, int64_t k, int64_t chunk,
                      double* __restrict__ part) {
  constexpr int W = kWarps;
  __shared__ double sums[W][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t rb = int64_t(blockIdx.x) * chunk, re = min(n, rb + chunk);
  double acc = 0.0;
  if (j < k) {
    const double th = theta[j];
    int64_t r = rb + w;
    for (; r + 3 * W < re; r += 4 * W) {           // four rows' loads in flight, added in order
      double d[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        d[q] = double(LX[(r + q * W) * k + j]) - th * double(X[(r + q * W) * k + j]);
#pragma unroll
      for (int q = 0; q < 4; ++q) acc = fma(d[q], d[q], acc);
    }
    for (; r < re; r += W) {
      const double d = double(LX[r * k + j]) - th * double(X[r * k + j]);
      acc = fma(d, d, acc);
    }
  }
  sums[w][lane] = acc;
  __syncthreads();
  if (w == 0 && j < k) {
    double s = 0.0;
    for (int q = 0; q < W; ++q) s += sums[q][lane];
    part[int64_t(blockIdx.x) * k + j] = s;
  }
}

template <typename T>
__global__ void block_random_kernel(int64_t count, uint64_t seed, T* __restrict__ X) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < count;
       i += int64_t(gridDim.x) * blockDim.x)
    X[i] = T(hash_uniform(seed, (uint64_t)i));
}

template <typename T, int MT>
int gram_mt(int64_t n, const T* A, int64_t ka, const T* B, int64_t kb, double* C, cudaStream_t st) {
  constexpr int TT = Tile<MT>::T, KS = Tile<MT>::KS;
  const int64_t ta = ceil_div(ka, TT), tb = ceil_div(kb, TT);
  GSP_REQUIRE(ta < 65536 && tb < 65536, "block too wide");
  // enough partitions to fill the GPU when the output is a few tiles, one when it is large: at
  // most kMaxParts for the widest micro tile, 2x / 4x as many for the narrower ones, whose CTAs
  // do less work and whose partials are smaller
  const int64_t parts = std::max<int64_t>(
      1, std::min<int64_t>(ceil_div(n, 8 * KS),
                           kMaxParts * (8 / MT) / std::min(ta * tb, kMaxParts * (8 / MT))));
  const int64_t chunk = ceil_div(ceil_div(n, parts), KS) * KS;
  const int64_t used = ceil_div(n, chunk);
  Scratch<double> parts_buf(st);
  if (used > 1) GSP_CUDA(parts_buf.alloc(used * ka * kb));
  double* part = used > 1 ? parts_buf.get() : C;
  dim3 grid((unsigned)used, (unsigned)ta, (unsigned)tb);
  block_gram_kernel<T, MT><<<grid, kBlockThreads, 0, st>>>(n, A, ka, B, kb, chunk, part);
  GSP_LAUNCH_CHECK("block_gram");
  return used > 1 ? sum_parts(part, used, ka * kb, C, st) : GSP_OK;
}

template <typename T>
int block_gram(int64_t n, const T* A, int64_t ka, const T* B, int64_t kb, double* C,
               cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && ka >= 1 && kb >= 1, "bad sizes");
  if (n == 0) {
    GSP_CUDA(cudaMemsetAsync(C, 0, ka * kb * sizeof(double), st));
    return GSP_OK;
  }
  switch (micro_tile(ka, kb)) {
    case 2: return gram_mt<T, 2>(n, A, ka, B, kb, C, st);
    case 4: return gram_mt<T, 4>(n, A, ka, B, kb, C, st);
    default: return gram_mt<T, 8>(n, A, ka, B, kb, C, st);
  }
}

template <typename T, int MT>
int combine_mt(int64_t n, const T* A, int64_t ka, const double* Q, int64_t kq, T* Y,
               cudaStream_t st) {
  constexpr int TT = Tile<MT>::T;
  const int64_t tr = ceil_div(n, TT), tq = ceil_div(kq, TT);
  GSP_REQUIRE(tr < (int64_t(1) << 31) && tq < 65536, "block too large");
  dim3 grid((unsigned)tr, (unsigned)tq);
  block_combine_kernel<T, MT><<<grid, kBlockThreads, 0, st>>>(n, A, ka, Q, kq, Y);
  GSP_LAUNCH_CHECK("block_combine");
  return GSP_OK;
}

template <typename T>
int block_combine(int64_t n, const T* A, int64_t ka, const double* Q, int64_t kq, T* Y,
                  cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && ka >= 1 && kq >= 1, "bad sizes");
  if (n == 0) return GSP_OK;
  switch (micro_tile(ka, kq)) {
    case 2: return combine_mt<T, 2>(n, A, ka, Q, kq, Y, st);
    case 4: return combine_mt<T, 4>(n, A, ka, Q, kq, Y, st);
    default: return combine_mt<T, 8>(n, A, ka, Q, kq, Y, st);
  }
}

template <typename T>
int block_residual(int64_t n, const T* X, const T* LX, const double* theta, int64_t k,
                   double* out, cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && k >= 1, "bad sizes");
  if (n == 0) {
    GSP_CUDA(cudaMemsetAsync(out, 0, k * sizeof(double), st));
    return GSP_OK;
  }
  const int64_t cg = ceil_div(k, 32);
  GSP_REQUIRE(cg < 65536, "block too wide");
  const Parts P = row_parts(n);
  Scratch<double> parts_buf(st);
  if (P.used > 1) GSP_CUDA(parts_buf.alloc(P.used * k));
  double* part = P.used > 1 ? parts_buf.get() : out;
  block_residual_kernel<T><<<dim3((unsigned)P.used, (unsigned)cg), kThreads, 0, st>>>(
      n, X, LX, theta, k, P.chunk, part);
  GSP_LAUNCH_CHECK("block_residual");
  return P.used > 1 ? sum_parts(part, P.used, k, out, st) : GSP_OK;
}

template <typename T>
int block_random(int64_t n, int64_t k, uint64_t seed, T* X, cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && k >= 1, "bad sizes");
  if (n == 0) return GSP_OK;
  block_random_kernel<T><<<grid_for(n * k), kThreads, 0, st>>>(n * k, seed, X);
  GSP_LAUNCH_CHECK("block_random");
  return GSP_OK;
}

}  // namespace

__global__ void sum_parts_kernel(int64_t count, int64_t parts, const double* __restrict__ part,
                                 double* __restrict__ out) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < count;
       e += int64_t(gridDim.x) * blockDim.x) {
    // loads issued eight at a time, added in p order
    double s = 0.0;
    int64_t p = 0;
    for (; p + 8 <= parts; p += 8) {
      double v[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) v[q] = part[(p + q) * count + e];
#pragma unroll
      for (int q = 0; q < 8; ++q) s += v[q];
    }
    for (; p < parts; ++p) s += part[p * count + e];
    out[e] = s;
  }
}

int sum_parts(const double* part, int64_t parts, int64_t count, double* out, cudaStream_t st) {
  sum_parts_kernel<<<grid_for(count), kThreads, 0, st>>>(count, parts, part, out);
  GSP_LAUNCH_CHECK("sum_parts");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {

#define GSP_BLOCK_API(SUF, T)                                                                      \
  int gsp_block_gram_##SUF(int64_t n, const T* A, int64_t ka, const T* B, int64_t kb, double* C,   \
                           void* stream) {                                                         \
    return gsp::block_gram<T>(n, A, ka, B, kb, C, gsp::as_stream(stream));                         \
  }                                                                                                \
  int gsp_block_combine_##SUF(int64_t n, const T* A, int64_t ka, const double* Q, int64_t kq,      \
                              T* Y, void* stream) {                                                \
    return gsp::block_combine<T>(n, A, ka, Q, kq, Y, gsp::as_stream(stream));                      \
  }                                                                                                \
  int gsp_block_residual_##SUF(int64_t n, const T* X, const T* LX, const double* theta, int64_t k, \
                               double* out, void* stream) {                                        \
    return gsp::block_residual<T>(n, X, LX, theta, k, out, gsp::as_stream(stream));                \
  }                                                                                                \
  int gsp_block_random_##SUF(int64_t n, int64_t k, uint64_t seed, T* X, void* stream) {            \
    return gsp::block_random<T>(n, k, seed, X, gsp::as_stream(stream));                            \
  }

GSP_BLOCK_API(f32, float)
GSP_BLOCK_API(f64, double)

}  // extern "C"
