// Fruchterman-Reingold spring layout (pygsp/graphs/_layout.py:169-219, DESIGN.md 4.14).
//
// One iteration of the reference moves every vertex i that is not fixed by
//
//   disp_i = sum_j delta_ij k^2 / d_ij^2  -  sum_{j : W_ij > 0} delta_ij d_ij / k,
//   delta_ij = p_i - p_j,  d_ij = max(|delta_ij|, 0.01),
//   length_i = |disp_i| (0.1 when below 0.01),  p_i += disp_i t / length_i.
//
// The repulsion is an all-pairs (n-body) sum in float64.  A CTA owns kQ = kThreads * kR query
// vertices, kept in registers (kR per thread), and one chunk of the candidate range; candidates
// are staged kTile at a time in shared memory (structure of arrays) and read by broadcast.  The
// self pair and duplicate points have delta = 0 and add exact zeros.  Each (chunk, vertex)
// partial goes to scratch; the update kernel adds the partials in chunk order, then the
// attraction over row i of W's CSR (entries with w > 0: the reference's A = W > 0, graph.py:718),
// and moves the vertex.  The chunk count depends on n only, so the result does not depend on the
// card, and no sum uses atomics: the same inputs give the same bits.  Positions ping-pong
// between two blocks because every CTA reads the previous state.
//
// 1/d^2 is MUFU.RCP64H refined by one cubic Newton step (three DFMA), accurate to a few ulp;
// d^2 is clamped at 0.01^2 before the reciprocal, which is the reference's clamp of d to within
// rounding, and k^2 multiplies each chunk's sum once.  That is 10 FP64 instructions per pair at
// dim = 2 (DESIGN.md 4.14).  Dimensions 1, 2 and 3 run the tiled kernel; any other dimension runs one generic
// kernel (one thread per vertex and chunk, partials accumulated in place) that is correct, not
// fast.
#include <math.h>

#include "common.cuh"
#include "gspb200.h"
#include "spring.cuh"

namespace gsp {
namespace {

constexpr int kThreads = 128;     // threads per CTA of the repulsion kernel
constexpr int kR = 4;             // query vertices per thread
constexpr int kQ = kThreads * kR; // query vertices per CTA
constexpr int kTile = 256;        // candidates staged in shared memory at a time
constexpr int kUnroll = 4;        // candidates per inner-loop trip
// CTAs the repulsion aims for (about 8 per SM of a 132-SM H100).  A constant, so that the chunk
// count below is a function of n alone.
constexpr int64_t kTargetCtas = 1056;
using spring::inv_d2;
using spring::spring_update_kernel;

struct Chunks {
  int64_t count, len;   // candidate range split into `count` chunks of `len` (a multiple of kTile)
};

Chunks chunks_for(int64_t n) {
  const int64_t qblocks = ceil_div(n, kQ);
  int64_t c = std::min(ceil_div(kTargetCtas, qblocks), ceil_div(n, kTile));
  c = std::max<int64_t>(c, 1);
  const int64_t len = ceil_div(ceil_div(n, c), kTile) * kTile;
  return {ceil_div(n, len), len};
}

// partial[c][i][:] = k^2 sum_{j in chunk c} delta_ij / d_ij^2 for dim = DIM (1, 2, 3)
template <int DIM>
__global__ void __launch_bounds__(kThreads)
    spring_repulsion_kernel(int64_t n, const double* __restrict__ pos, double k2, int64_t chunk_len,
                            double* __restrict__ partial) {
  __shared__ double sc[DIM][kTile];
  const int64_t q0 = int64_t(blockIdx.x) * kQ;
  const int64_t c0 = int64_t(blockIdx.y) * chunk_len;
  const int64_t c1 = min(n, c0 + chunk_len);

  double q[kR][DIM], acc[kR][DIM];
#pragma unroll
  for (int r = 0; r < kR; ++r) {
    const int64_t i = q0 + threadIdx.x + r * kThreads;
#pragma unroll
    for (int a = 0; a < DIM; ++a) {
      q[r][a] = i < n ? pos[i * DIM + a] : 0.0;
      acc[r][a] = 0.0;
    }
  }

  for (int64_t t0 = c0; t0 < c1; t0 += kTile) {
    const int cn = int(min(int64_t(kTile), c1 - t0));
    __syncthreads();   // the previous tile is consumed
    for (int e = threadIdx.x; e < cn * DIM; e += kThreads) {
      const int j = e / DIM;
      sc[e - j * DIM][j] = pos[t0 * DIM + e];
    }
    __syncthreads();
    int j = 0;
    for (; j + kUnroll <= cn; j += kUnroll) {
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        double c[DIM];
#pragma unroll
        for (int a = 0; a < DIM; ++a) c[a] = sc[a][j + u];
#pragma unroll
        for (int r = 0; r < kR; ++r) {
          double dl[DIM];
          double d2 = 0.0;
#pragma unroll
          for (int a = 0; a < DIM; ++a) {
            dl[a] = q[r][a] - c[a];
            d2 = a == 0 ? dl[a] * dl[a] : fma(dl[a], dl[a], d2);
          }
          const double f = inv_d2(d2);
#pragma unroll
          for (int a = 0; a < DIM; ++a) acc[r][a] = fma(dl[a], f, acc[r][a]);
        }
      }
    }
    for (; j < cn; ++j) {
      double c[DIM];
#pragma unroll
      for (int a = 0; a < DIM; ++a) c[a] = sc[a][j];
#pragma unroll
      for (int r = 0; r < kR; ++r) {
        double dl[DIM];
        double d2 = 0.0;
#pragma unroll
        for (int a = 0; a < DIM; ++a) {
          dl[a] = q[r][a] - c[a];
          d2 = a == 0 ? dl[a] * dl[a] : fma(dl[a], dl[a], d2);
        }
        const double f = inv_d2(d2);
#pragma unroll
        for (int a = 0; a < DIM; ++a) acc[r][a] = fma(dl[a], f, acc[r][a]);
      }
    }
  }

  double* out = partial + int64_t(blockIdx.y) * n * DIM;
#pragma unroll
  for (int r = 0; r < kR; ++r) {
    const int64_t i = q0 + threadIdx.x + r * kThreads;
    if (i < n) {
#pragma unroll
      for (int a = 0; a < DIM; ++a) out[i * DIM + a] = k2 * acc[r][a];
    }
  }
}

// the same sum for any dim: one thread per (vertex, chunk), accumulated in place in `partial`
__global__ void spring_repulsion_generic_kernel(int64_t n, int dim, const double* __restrict__ pos,
                                                double k2, int64_t chunk_len, double* partial) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t c0 = int64_t(blockIdx.y) * chunk_len;
  const int64_t c1 = min(n, c0 + chunk_len);
  const double* p = pos + i * dim;
  double* out = partial + (int64_t(blockIdx.y) * n + i) * dim;
  for (int a = 0; a < dim; ++a) out[a] = 0.0;
  for (int64_t j = c0; j < c1; ++j) {
    const double* c = pos + j * dim;
    double d2 = 0.0;
    for (int a = 0; a < dim; ++a) {
      const double dl = p[a] - c[a];
      d2 = a == 0 ? dl * dl : fma(dl, dl, d2);
    }
    const double f = inv_d2(d2);
    for (int a = 0; a < dim; ++a) out[a] = fma(p[a] - c[a], f, out[a]);
  }
  for (int a = 0; a < dim; ++a) out[a] *= k2;
}

template <typename T>
int spring_step(int64_t n, int dim, const int32_t* indptr, const int32_t* indices, const T* data,
                double k, double t, const uint8_t* fixed, const double* pos_in, double* pos_out,
                const Chunks& ch, double* partial, cudaStream_t st) {
  const double k2 = k * k;
  const dim3 grid((unsigned)ceil_div(n, kQ), (unsigned)ch.count);
  if (dim == 1) {
    spring_repulsion_kernel<1><<<grid, kThreads, 0, st>>>(n, pos_in, k2, ch.len, partial);
  } else if (dim == 2) {
    spring_repulsion_kernel<2><<<grid, kThreads, 0, st>>>(n, pos_in, k2, ch.len, partial);
  } else if (dim == 3) {
    spring_repulsion_kernel<3><<<grid, kThreads, 0, st>>>(n, pos_in, k2, ch.len, partial);
  } else {
    const dim3 generic((unsigned)ceil_div(n, 128), (unsigned)ch.count);
    spring_repulsion_generic_kernel<<<generic, 128, 0, st>>>(n, dim, pos_in, k2, ch.len, partial);
  }
  GSP_LAUNCH_CHECK("spring_repulsion");
  spring_update_kernel<T><<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(
      n, dim, indptr, indices, data, k, t, fixed, ch.count, pos_in, partial, pos_out);
  GSP_LAUNCH_CHECK("spring_update");
  return GSP_OK;
}

#define GSP_REQUIRE_SPRING(n, dim, pos)                                                         \
  GSP_REQUIRE((n) >= 0 && (n) < (int64_t(1) << 31), "bad vertex count");                        \
  GSP_REQUIRE((dim) >= 1 && int64_t(dim) * (n) < (int64_t(1) << 40), "bad layout dimension");   \
  GSP_REQUIRE((n) == 0 || (pos) != nullptr, "positions are NULL")

template <typename T>
int spring_step_api(int64_t n, int dim, const int32_t* indptr, const int32_t* indices,
                    const T* data, double k, double t, const uint8_t* fixed, const double* pos_in,
                    double* pos_out, cudaStream_t st) {
  GSP_REQUIRE_SPRING(n, dim, pos_in);
  GSP_REQUIRE(n == 0 || (pos_out != nullptr && pos_out != pos_in),
              "pos_out must be a distinct block");
  if (n == 0) return GSP_OK;
  const Chunks ch = chunks_for(n);
  Scratch<double> partial(st);
  GSP_CUDA(partial.alloc(size_t(ch.count) * n * dim));
  return spring_step<T>(n, dim, indptr, indices, data, k, t, fixed, pos_in, pos_out, ch,
                        partial.get(), st);
}

template <typename T>
int spring_layout(int64_t n, int dim, const int32_t* indptr, const int32_t* indices,
                  const T* data, double k, int iterations, const double* temps_host,
                  const uint8_t* fixed, double* pos, double* states, cudaStream_t st) {
  GSP_REQUIRE_SPRING(n, dim, pos);
  GSP_REQUIRE(iterations >= 0, "iterations must be >= 0");
  GSP_REQUIRE(iterations == 0 || temps_host != nullptr, "temperatures are NULL");
  if (n == 0 || iterations == 0) return GSP_OK;
  const size_t block = size_t(n) * dim;
  const Chunks ch = chunks_for(n);
  Scratch<double> partial(st);
  GSP_CUDA(partial.alloc(size_t(ch.count) * block));
  // with `states`, iteration it writes states[it]; otherwise pos and one scratch block alternate
  Scratch<double> other(st);
  if (states == nullptr) GSP_CUDA(other.alloc(block));
  const double* cur = pos;
  for (int it = 0; it < iterations; ++it) {
    double* next = states != nullptr ? states + it * block : (it % 2 == 0 ? other.get() : pos);
    const int rc = spring_step<T>(n, dim, indptr, indices, data, k, temps_host[it], fixed, cur,
                                  next, ch, partial.get(), st);
    if (rc != GSP_OK) return rc;
    cur = next;
  }
  if (cur != pos)
    GSP_CUDA(cudaMemcpyAsync(pos, cur, block * sizeof(double), cudaMemcpyDeviceToDevice, st));
  return GSP_OK;
}

}  // namespace
}  // namespace gsp

extern "C" {

#define GSP_LAYOUT_API(SUF, T)                                                                  \
  int gsp_spring_step_##SUF(int64_t n, int dim, const int32_t* indptr, const int32_t* indices,   \
                            const T* data, double k, double t, const uint8_t* fixed,            \
                            const double* pos_in, double* pos_out, void* stream) {              \
    return gsp::spring_step_api<T>(n, dim, indptr, indices, data, k, t, fixed, pos_in, pos_out, \
                                   gsp::as_stream(stream));                                     \
  }                                                                                             \
  int gsp_spring_layout_##SUF(int64_t n, int dim, const int32_t* indptr, const int32_t* indices, \
                              const T* data, double k, int iterations, const double* temps_host, \
                              const uint8_t* fixed, double* pos, double* states, void* stream) { \
    return gsp::spring_layout<T>(n, dim, indptr, indices, data, k, iterations, temps_host, fixed, \
                                 pos, states, gsp::as_stream(stream));                          \
  }

GSP_LAYOUT_API(f32, float)
GSP_LAYOUT_API(f64, double)

}  // extern "C"
