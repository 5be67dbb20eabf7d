// Fixed-order reductions: the summation order behind every bit-reproducible device solver.
//
// Column sums over rows (csrc/block.cu, csrc/krylov.cu, csrc/moments.cu) are two-level.
// row_parts splits the n rows into min(ceil(n / 1024), kMaxParts) parts of ceil(n / parts) rows
// (the last may be shorter), a function of n alone: parts are at most 1024 rows up to
// kMaxParts * 1024 rows and longer only past it (n = 1025 gives two parts of 513 rows,
// n = 263 * 1024 + 1 gives 264 parts of 1021); CTA p sums part p with column_part (lane =
// column, warp w takes rows w, w + 8, ... in order, the warp sums are added in warp order) and
// sum_parts adds the partials in p order.  So a column's bits do not depend on the other
// columns, on how many there are or on the device.
// csrc/cg.cu forms its own per-CTA partials and adds them with sum_parts.
//
// A FISTA pass (csrc/simplex.cu, csrc/tv.cu) is one launch of pass_blocks CTAs whose last CTA to
// finish adds the CTA partials (fista_last_block) and applies the solver's stop rule; the solver's
// scratch has the kFista* layout.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {

constexpr int kThreads = 256;     // threads per CTA of every pass below
constexpr int kWarps = kThreads / 32;
// Row partitions of a column reduction: at most this many partials per column (two CTAs per SM
// of an H100).  Constants, so that the summation order -- and hence the result -- is the same on
// every device.
constexpr int64_t kMaxParts = 264;

struct Parts {
  int64_t used, chunk;
};

// the row partition of a column reduction over n >= 1 rows: part p is rows [p chunk, (p+1) chunk)
inline Parts row_parts(int64_t n) {
  const int64_t parts = std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, 1024), kMaxParts));
  const int64_t chunk = ceil_div(n, parts);
  return {ceil_div(n, chunk), chunk};
}

// grid of a grid-stride pass of kThreads-thread CTAs over count items
inline int grid_for(int64_t count) {
  return (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(count, kThreads), 4096));
}

// grid of a pass that strides over n items, rpb per block: four blocks per SM at most, and at most
// max_blocks (the size of the caller's per-block partials area)
static inline int pass_blocks(int64_t n, int rpb, int max_blocks) {
  return (int)std::max<int64_t>(
      1, std::min<int64_t>(ceil_div(n, rpb), std::min<int64_t>(int64_t(sm_count()) * 4, max_blocks)));
}

// sum over the w lanes of an aligned power-of-two sub-warp (xor butterfly: fixed order)
template <typename S>
__device__ __forceinline__ S group_sum(S v, int w) {
  for (int off = w >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// The CTA's partial of one per-column sum.  Lane = column, warp w holds in acc its sum over rows
// w, w + 8, ...; the warp sums are added in warp order and warp 0 writes its column's to *out
// where valid (the column exists).  Every thread of the CTA calls it.  block_residual_kernel
// (csrc/block.cu) and moments_part_kernel (csrc/moments.cu) add in this order by hand: through
// this helper nvcc schedules their row loops' loads less deeply, and the moments pass ran 12%
// slower on an H100.
__device__ __forceinline__ void column_part(double acc, bool valid, double* out) {
  __shared__ double sums[kWarps][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  sums[w][lane] = acc;
  __syncthreads();
  if (w == 0 && valid) {
    double s = 0.0;
    for (int k = 0; k < kWarps; ++k) s += sums[k][lane];
    *out = s;
  }
}

// out[e] = sum_{p < parts} part[p * count + e], p in order: the second level of a column reduction
// (csrc/block.cu)
int sum_parts(const double* part, int64_t parts, int64_t count, double* out, cudaStream_t st);

// Scratch of a FISTA solver, in doubles: [0] t_k, [1] the stop criterion (0 = running), [2] the
// stop iteration, [3] the arrival counter (uint64 bits); from kFistaPart the CTA partials of up to
// kFistaSums sums, from kFistaHistory the history the host reads.
constexpr int kFistaMaxBlocks = 1024;
constexpr int kFistaSums = 3;
constexpr int kFistaPart = 8;
constexpr int kFistaHistory = kFistaPart + kFistaSums * kFistaMaxBlocks;
static_assert(GSPB200_FB_HISTORY == kFistaHistory && GSPB200_TV_HISTORY == kFistaHistory,
              "FISTA scratch layout");

// End of a FISTA pass of kThreads-thread CTAs.  The CTA's partial of each of the Q sums in v
// (warp butterflies, then the warps in order) goes to the partials area of scal.  The last CTA to
// arrive re-arms the arrival counter and adds the partials over the CTAs (warp q takes sum q:
// lanes strided over the CTAs, then a butterfly -- a fixed order for a given grid); its thread 0
// then calls last(tot) with the Q totals.  Every thread of the CTA calls it.
template <int Q, typename F>
__device__ __forceinline__ void fista_last_block(const double (&v)[Q], double* scal, F&& last) {
  static_assert(Q <= kFistaSums, "FISTA partials area");
  __shared__ double sh[Q][kWarps];
  __shared__ bool is_last;
  const int warp = threadIdx.x / 32, wl = threadIdx.x % 32;
  double s[Q];
#pragma unroll
  for (int q = 0; q < Q; ++q) s[q] = group_sum(v[q], 32);
  if (wl == 0)
#pragma unroll
    for (int q = 0; q < Q; ++q) sh[q][warp] = s[q];
  __syncthreads();
  double* part = scal + kFistaPart;
  if (threadIdx.x < Q) {
    double acc = 0;
    for (int k = 0; k < kWarps; ++k) acc += sh[threadIdx.x][k];
    part[int64_t(blockIdx.x) * Q + threadIdx.x] = acc;
    __threadfence();
  }
  __syncthreads();
  unsigned long long* counter = reinterpret_cast<unsigned long long*>(scal) + 3;
  if (threadIdx.x == 0) is_last = atomicAdd(counter, 1ull) == (unsigned long long)(gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (warp < Q) {
    double acc = 0;
    for (int b = wl; b < int(gridDim.x); b += 32) acc += __ldcg(part + int64_t(b) * Q + warp);
    acc = group_sum(acc, 32);
    if (wl == 0) sh[warp][0] = acc;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *counter = 0ull;                               // every CTA has arrived: ready for the next pass
    double tot[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) tot[q] = sh[q][0];
    last(tot);
  }
}

// Lanes of a FISTA pass over rows of `cols` values: for cols <= 32 a sub-warp of w =
// 2^ceil(log2 cols) lanes per row and V = 1 value per lane; wider rows a warp (w = 32) with V
// values per lane, the power of two that covers cols / 32 but at most 8 (wider rows go in chunks
// of 32 V).
struct Lanes {
  int w, V;
};

inline Lanes fista_lanes(int cols) {
  Lanes l{1, 1};
  if (cols <= 32) {
    while (l.w < cols) l.w *= 2;
  } else {
    l.w = 32;
    while (32 * l.V < cols && l.V < 8) l.V *= 2;
  }
  return l;
}

// launch(std::integral_constant<int, V>()) for V = l.V: the kernel instance for those lanes
template <typename F>
int launch_lanes(const Lanes& l, F&& launch) {
  switch (l.V) {
    case 1: return launch(std::integral_constant<int, 1>());
    case 2: return launch(std::integral_constant<int, 2>());
    case 4: return launch(std::integral_constant<int, 4>());
    default: return launch(std::integral_constant<int, 8>());
  }
}

}  // namespace gsp
