// Effective resistances of graph_sparsify past the dense factor (pygsp/reduction.py:84, :101):
// the Johnson-Lindenstrauss sketch of Spielman-Srivastava (Theorem 2 of "Graph sparsification by
// effective resistances"), R~_e = ||Z (chi_u - chi_v)||^2 with Z = Q W^1/2 B L^+ / sqrt(k).
//
// The caller solves the Jacobi-scaled system Lhat U = Y, Lhat = D^-1/2 L D^-1/2, by block CG
// (csrc/cg.cu) for blocks of columns j0 .. j0 + width - 1 of the k columns, and Z = D^-1/2 U.
//
//   gsp_jl_sketch_f64       Y[i][c] = dinv[i] / sqrt(k) * sum over the stored off-diagonal entries
//                           (i, v) of row i, in CSR order, of s(i, v) sqrt(-L_iv) q_j({i, v}),
//                           j = j0 + c: the block of D^-1/2 B^T W^1/2 Q^T / sqrt(k).  s = +1 when i
//                           is the larger end of the edge, else -1 (the incidence matrix B).
//   gsp_jl_accumulate_f64   R[e] += sum_c (dinv[u] U[u][c] - dinv[v] U[v][c])^2 for u = erow[e],
//                           v = ecol[e]: the block's share of R~_e, columns in a fixed order.
//
// Signs.  Edge {a < b} and column j: q_j = +1 when bit (j mod 128) of the 128 bits of
// curand4(curand_init(key, a n + b, 4 (j div 128))) is 0, else -1, where bit t is bit (t mod 32)
// of word t div 32 of (x, y, z, w).  Both ends of an edge recompute the same draw, so nothing is
// stored and nothing is added atomically; one Philox block serves 128 columns of one entry.
//
// Mapping.  Sketch: one warp per row; lane l owns the block's columns l + 32 r (r < 8).  The row's
// entries go 32 at a time: lane m of the warp draws the Philox blocks of entry m (at most three:
// 256 columns starting anywhere), and every lane reads the words it needs by shuffles.
// Accumulate: one warp per edge, lanes over columns, a fixed butterfly over the lanes.  Both are
// bit-reproducible; neither allocates.
#include <curand_kernel.h>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxWidth = 256;
constexpr int kMaxCols = kMaxWidth / 32;   // columns per lane
constexpr int kMaxDraws = 3;               // Philox blocks spanned by 256 consecutive columns

__device__ __forceinline__ uint4 draw4(uint64_t key, uint64_t sub, uint64_t t) {
  curandStatePhilox4_32_10_t state;
  curand_init(key, sub, 4ull * t, &state);
  return curand4(&state);
}

__global__ void __launch_bounds__(kThreads)
jl_sketch_kernel(int64_t n, const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                 const double* __restrict__ data, const double* __restrict__ dinv, uint64_t key,
                 int64_t j0, int width, double scale, double* __restrict__ Y) {
  const int lane = threadIdx.x & 31;
  const int64_t i = int64_t(blockIdx.x) * kWarps + (threadIdx.x >> 5);
  if (i >= n) return;                                   // whole warps leave together
  const int64_t t0 = j0 >> 7;
  const int nt = int(((j0 + width - 1) >> 7) - t0) + 1;
  // per owned column: which Philox block, which word and which bit it reads
  int tr[kMaxCols], wr[kMaxCols];
  const int sh = int((j0 + lane) & 31);
#pragma unroll
  for (int r = 0; r < kMaxCols; ++r) {
    const int64_t j = j0 + lane + 32 * r;
    tr[r] = int((j >> 7) - t0);
    wr[r] = int((j >> 5) & 3);
  }
  double acc[kMaxCols];
#pragma unroll
  for (int r = 0; r < kMaxCols; ++r) acc[r] = 0.0;

  const int64_t b = indptr[i], e = indptr[i + 1];
  for (int64_t base = b; base < e; base += 32) {
    const int cnt = e - base < 32 ? int(e - base) : 32;
    double val = 0.0;
    uint4 d[kMaxDraws] = {};
    if (lane < cnt) {
      const int64_t v = indices[base + lane];
      const double w = -data[base + lane];
      if (v != i) {
        val = i > v ? sqrt(w) : -sqrt(w);
        const uint64_t a = uint64_t(i < v ? i : v), c = uint64_t(i < v ? v : i);
        const uint64_t sub = a * uint64_t(n) + c;
#pragma unroll
        for (int t = 0; t < kMaxDraws; ++t)
          if (t < nt) d[t] = draw4(key, sub, uint64_t(t0 + t));
      }
    }
    for (int m = 0; m < cnt; ++m) {
      const double vm = __shfl_sync(0xffffffffu, val, m);
      uint32_t neg[kMaxCols];
#pragma unroll
      for (int r = 0; r < kMaxCols; ++r) neg[r] = 0;
#pragma unroll
      for (int t = 0; t < kMaxDraws; ++t) {
        if (t < nt) {
          const uint32_t x = __shfl_sync(0xffffffffu, d[t].x, m);
          const uint32_t y = __shfl_sync(0xffffffffu, d[t].y, m);
          const uint32_t z = __shfl_sync(0xffffffffu, d[t].z, m);
          const uint32_t ww = __shfl_sync(0xffffffffu, d[t].w, m);
#pragma unroll
          for (int r = 0; r < kMaxCols; ++r) {
            const uint32_t word = wr[r] == 0 ? x : wr[r] == 1 ? y : wr[r] == 2 ? z : ww;
            if (tr[r] == t) neg[r] = (word >> sh) & 1u;
          }
        }
      }
#pragma unroll
      for (int r = 0; r < kMaxCols; ++r) acc[r] += neg[r] ? -vm : vm;
    }
  }
  const double s = dinv[i] * scale;
#pragma unroll
  for (int r = 0; r < kMaxCols; ++r) {
    const int c = lane + 32 * r;
    if (c < width) Y[i * width + c] = acc[r] * s;
  }
}

__global__ void __launch_bounds__(kThreads)
jl_accumulate_kernel(int64_t ne, const int32_t* __restrict__ erow, const int32_t* __restrict__ ecol,
                     const double* __restrict__ U, const double* __restrict__ dinv, int width,
                     double* __restrict__ R) {
  const int lane = threadIdx.x & 31;
  const int64_t e = int64_t(blockIdx.x) * kWarps + (threadIdx.x >> 5);
  if (e >= ne) return;
  const int64_t u = erow[e], v = ecol[e];
  const double du = dinv[u], dv = dinv[v];
  const double* Uu = U + u * width;
  const double* Uv = U + v * width;
  double acc = 0.0;
  for (int c = lane; c < width; c += 32) {
    const double z = du * Uu[c] - dv * Uv[c];
    acc += z * z;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if (lane == 0) R[e] += acc;
}

}  // namespace

int jl_sketch(int64_t n, const int32_t* indptr, const int32_t* indices, const double* data,
              const double* dinv, uint64_t key, int64_t j0, int width, int64_t k, double* Y,
              cudaStream_t st) {
  if (n == 0) return GSP_OK;
  jl_sketch_kernel<<<(unsigned)ceil_div(n, kWarps), kThreads, 0, st>>>(
      n, indptr, indices, data, dinv, key, j0, width, 1.0 / sqrt(double(k)), Y);
  GSP_LAUNCH_CHECK("jl_sketch");
  return GSP_OK;
}

int jl_accumulate(int64_t ne, const int32_t* erow, const int32_t* ecol, const double* U,
                  const double* dinv, int width, double* R, cudaStream_t st) {
  if (ne == 0) return GSP_OK;
  jl_accumulate_kernel<<<(unsigned)ceil_div(ne, kWarps), kThreads, 0, st>>>(ne, erow, ecol, U,
                                                                           dinv, width, R);
  GSP_LAUNCH_CHECK("jl_accumulate");
  return GSP_OK;
}

}  // namespace gsp

extern "C" {
int gsp_jl_sketch_f64(int64_t n, const int32_t* indptr, const int32_t* indices, const double* data,
                      const double* dinv, uint64_t key, int64_t j0, int64_t width, int64_t k,
                      double* Y, void* stream) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31) && width >= 1 && width <= gsp::kMaxWidth &&
                  j0 >= 0 && k >= 1 && j0 + width <= k,
              "bad arguments");
  GSP_REQUIRE(n == 0 || (indptr && indices && data && dinv && Y), "no buffer");
  return gsp::jl_sketch(n, indptr, indices, data, dinv, key, j0, (int)width, k, Y,
                        gsp::as_stream(stream));
}
int gsp_jl_accumulate_f64(int64_t ne, const int32_t* erow, const int32_t* ecol, const double* U,
                          const double* dinv, int64_t width, double* R, void* stream) {
  GSP_REQUIRE(ne >= 0 && width >= 1 && width <= gsp::kMaxWidth, "bad arguments");
  GSP_REQUIRE(ne == 0 || (erow && ecol && U && dinv && R), "no buffer");
  return gsp::jl_accumulate(ne, erow, ecol, U, dinv, (int)width, R, gsp::as_stream(stream));
}
}
