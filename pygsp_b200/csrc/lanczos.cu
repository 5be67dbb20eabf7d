// Device Lanczos for Graph.estimate_lmax (pygsp/graphs/graph.py:858-931).
//
// Replaces ARPACK's dsaupd/dseupd reached through scipy.sparse.linalg.eigsh
// (graph.py:911-917): a three-term Lanczos recurrence whose operator is the
// same CSR SpMV kernel family as the filter, with the scalar recurrence
// coefficients kept ON DEVICE so that a whole batch of iterations is enqueued
// without a host round trip.  The host only reads the (alpha, beta) arrays
// back to diagonalise the small tridiagonal matrix and test convergence
// (|beta_m s_m| <= tol |theta|, ARPACK's criterion with tol = 5e-3).
#include "common.cuh"
#include "gspb200.h"

namespace gsp {

constexpr int kVecThreads = 256;
constexpr int kMaxVecBlocks = 2048;   // partial sums per reduction (scal_dev layout)

// sum over the block, returned to every thread; safe to call repeatedly
__device__ __forceinline__ double block_allreduce(double v) {
  __shared__ double part[kVecThreads / 32];
  __shared__ double total;
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    double s = threadIdx.x < kVecThreads / 32 ? part[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) total = s;
  }
  __syncthreads();
  const double out = total;
  __syncthreads();
  return out;
}

// Reductions are two-level and ORDER-FIXED (no floating-point atomics): every
// block writes one partial, every consumer block re-adds the partials in the
// same order, so a run is bit-reproducible.
__device__ __forceinline__ double sum_partials(const double* part, int count) {
  double acc = 0;
  for (int i = threadIdx.x; i < count; i += kVecThreads) acc += part[i];
  return block_allreduce(acc);
}

// counter-based generator: the start vector depends only on (seed, index)
__device__ __forceinline__ double hash_uniform(uint64_t seed, uint64_t i) {
  uint64_t z = seed + 0x9E3779B97F4A7C15ull * (i + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return double(z >> 11) * (1.0 / 9007199254740992.0) * 2.0 - 1.0;
}

template <typename T>
__global__ void lanczos_seed_kernel(int64_t n, T* v, uint64_t seed, double* part_out) {
  double acc = 0;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    const T x = T(hash_uniform(seed, (uint64_t)i));
    v[i] = x;
    acc += double(x) * double(x);
  }
  acc = block_allreduce(acc);
  if (threadIdx.x == 0) part_out[blockIdx.x] = acc;
}

// ------------------------------------------------------------------ SpMV
// y = scale * (A x), LPR lanes per row (LPR = the power of two >= the mean row length, 2..32,
// so that a row is normally ONE coalesced read of its entries and neighbouring rows' entries
// -- neighbours in memory -- share 128-byte lines), row sums reduced with warp shuffles
// (graph.py:911-917 spends its time in exactly this product).
//
// What bounds a thread-per-row or warp-per-row product on such graphs is not DRAM but the L1
// tag stage: a warp's 32 scalar gathers x[col] touch ~16 different lines.  So a
// block owns a TILE of TR consecutive rows and keeps x[tile] and indptr[tile] in shared
// memory: with a locality-preserving vertex numbering (Morton) ~90 % of a row's neighbours
// lie inside its own tile and are served from shared memory (conflict-limited, a few cycles per
// warp); the others take the global path.  U rows per lane group are in flight at once (a row
// is a dependent chain entry -> x[col]).
//
// Optionally the kernel leaves, per block, the partial sum of y_i * (scale * x_i): the Lanczos
// alpha = v' L v comes out of the same pass.  scale = 1 / sqrt(sum(inv_norm2_parts)) when
// inv_norm2_parts is given (x is then the unnormalised Lanczos vector u_j), else 1.
constexpr int kSpmvTileRows = 1024;

template <typename T, int LPR>
__global__ void __launch_bounds__(kVecThreads)
spmv_window_kernel(int64_t n, const int32_t* __restrict__ indptr,
                   const int32_t* __restrict__ indices, const T* __restrict__ vals,
                   const T* __restrict__ x, T* __restrict__ y, const double* norm2_parts,
                   int n_parts, double* beta_out, double* dot_parts, int tile_rows) {
  __shared__ T xs[kSpmvTileRows];
  __shared__ int32_t ps[kSpmvTileRows + 1];
  double scale = 1.0;
  if (norm2_parts) {
    const double nb = sqrt(sum_partials(norm2_parts, n_parts));
    scale = nb > 0 ? 1.0 / nb : 0.0;
    if (beta_out && blockIdx.x == 0 && threadIdx.x == 0) *beta_out = nb;
  }
  constexpr int RPB = kVecThreads / LPR;          // rows per block and pass
  constexpr int U = 4;                            // independent rows per lane group and trip
  const int lane = threadIdx.x % LPR;
  const int sub = threadIdx.x / LPR;
  double dot = 0;
  const int64_t n_tiles = (n + tile_rows - 1) / tile_rows;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int64_t r0 = tile * tile_rows;
    const int rows = (n - r0 < int64_t(tile_rows)) ? int(n - r0) : tile_rows;
    __syncthreads();                               // the previous tile's window is no longer read
    for (int i = threadIdx.x; i <= rows; i += kVecThreads) {
      ps[i] = __ldg(indptr + r0 + i);
      if (i < rows) xs[i] = __ldg(x + r0 + i);
    }
    __syncthreads();
    for (int base = 0; base < rows; base += RPB * U) {   // uniform trip count over the block
      double acc[U];
      int jn[U], je[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {                // first entry of U rows: loads issued together
        const int lr = base + u * RPB + sub;
        acc[u] = 0;
        jn[u] = je[u] = 0;
        int col = -1;
        T val = T(0);
        if (lr < rows) {
          const int j = ps[lr] + lane;
          je[u] = ps[lr + 1];
          jn[u] = j + LPR;
          if (j < je[u]) {
            col = __ldg(indices + j);
            val = __ldg(vals + j);
          }
        }
        if (col >= 0) {
          const unsigned off = unsigned(col - int(r0));   // int: n < 2^31 rows per block of L
          const T xv = (int64_t(col) >= r0 && off < unsigned(rows)) ? xs[off] : __ldg(x + col);
          acc[u] = double(val) * double(xv);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {                // rows longer than LPR entries
        for (int j = jn[u]; j < je[u]; j += LPR) {
          const int col = __ldg(indices + j);
          const unsigned off = unsigned(col - int(r0));
          const T xv = (int64_t(col) >= r0 && off < unsigned(rows)) ? xs[off] : __ldg(x + col);
          acc[u] += double(__ldg(vals + j)) * double(xv);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        double a = acc[u];
#pragma unroll
        for (int o = LPR / 2; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o, LPR);
        const int lr = base + u * RPB + sub;
        if (lr < rows && lane == 0) {
          const double yi = a * scale;
          y[r0 + lr] = T(yi);
          if (dot_parts) dot += double(T(yi)) * (double(xs[lr]) * scale);
        }
      }
    }
  }
  if (dot_parts) {                                 // uniform branch
    dot = block_allreduce(dot);
    if (threadIdx.x == 0) dot_parts[blockIdx.x] = dot;
  }
}

// The first form of the product (no shared-memory window): LPR = the largest power of two <=
// the mean row length, every lane group walks its row in steps of LPR.  Kept selectable
// (GSPB200_SPMV=subwarp) for A/B measurements and for numberings without locality.
template <typename T, int LPR>
__global__ void __launch_bounds__(kVecThreads)
spmv_subwarp_kernel(int64_t n, const int32_t* __restrict__ indptr,
                    const int32_t* __restrict__ indices, const T* __restrict__ vals,
                    const T* __restrict__ x, T* __restrict__ y, const double* norm2_parts,
                    int n_parts, double* beta_out, double* dot_parts) {
  double scale = 1.0;
  if (norm2_parts) {
    const double nb = sqrt(sum_partials(norm2_parts, n_parts));
    scale = nb > 0 ? 1.0 / nb : 0.0;
    if (beta_out && blockIdx.x == 0 && threadIdx.x == 0) *beta_out = nb;
  }
  constexpr int RPB = kVecThreads / LPR;          // rows per block and pass
  constexpr int U = 4;                            // independent rows per lane group and trip:
  const int lane = threadIdx.x % LPR;             // a row is three dependent loads (indptr ->
  const int sub = threadIdx.x / LPR;              // entry -> x[col]); U of them are in flight
  double dot = 0;
  for (int64_t base = int64_t(blockIdx.x) * (RPB * U); base < n;
       base += int64_t(gridDim.x) * (RPB * U)) {   // the trip count is uniform over the block
    int start[U], end[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t row = base + u * RPB + sub;
      start[u] = end[u] = 0;
      if (row < n) {
        start[u] = __ldg(indptr + row);
        end[u] = __ldg(indptr + row + 1);
      }
    }
    double acc[U];
    int col[U];
    T val[U];
    int more = 0;
#pragma unroll
    for (int u = 0; u < U; ++u) {                   // first entry of every row: loads issued together
      acc[u] = 0;
      const int j = start[u] + lane;
      const bool ok = j < end[u];
      col[u] = ok ? __ldg(indices + j) : -1;
      val[u] = ok ? __ldg(vals + j) : T(0);
      more |= (j + LPR < end[u]);
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
      if (col[u] >= 0) acc[u] = double(val[u]) * double(__ldg(x + col[u]));
    if (__any_sync(0xffffffffu, more)) {            // rows longer than LPR entries
#pragma unroll
      for (int u = 0; u < U; ++u)
        for (int j = start[u] + lane + LPR; j < end[u]; j += LPR)
          acc[u] += double(__ldg(vals + j)) * double(__ldg(x + __ldg(indices + j)));
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      double a = acc[u];
#pragma unroll
      for (int o = LPR / 2; o > 0; o >>= 1) a += __shfl_down_sync(0xffffffffu, a, o, LPR);
      const int64_t row = base + u * RPB + sub;
      if (row < n && lane == 0) {
        const double yi = a * scale;
        y[row] = T(yi);
        if (dot_parts) dot += double(T(yi)) * (double(x[row]) * scale);
      }
    }
  }
  if (dot_parts) {                                 // uniform branch
    dot = block_allreduce(dot);
    if (threadIdx.x == 0) dot_parts[blockIdx.x] = dot;
  }
}

static inline int spmv_lanes_subwarp(int64_t n, int64_t nnz) {
  const char* e = getenv("GSPB200_SPMV_LPR");
  if (e && (atoi(e) == 2 || atoi(e) == 4 || atoi(e) == 8 || atoi(e) == 16 || atoi(e) == 32))
    return atoi(e);
  // about three entries per lane: fewer, longer lane chains and more rows in flight per warp beat
  // one entry per lane (N = 1e6, 12.4 entries per row, L2-warm on an H100 SXM at 400 W: 4 lanes
  // 55-58 us, 16 lanes 70 us per product; tools/spmv_probe.py)
  const double mean = n > 0 ? double(nnz) / double(n) : 1.0;
  int lpr = 2;
  while (lpr < 32 && 3 * (2 * lpr) <= mean) lpr *= 2;
  return lpr;
}

static inline int spmv_lanes(int64_t n, int64_t nnz) {
  const double mean = n > 0 ? double(nnz) / double(n) : 1.0;
  int lpr = 2;
  while (lpr < 32 && lpr < mean) lpr *= 2;           // smallest power of two >= mean, in [2, 32]
  return lpr;
}

// rows per tile: up to kSpmvTileRows, smaller when the matrix would otherwise leave SMs idle
static inline int spmv_tile_rows(int64_t n) {
  const char* e = getenv("GSPB200_SPMV_TR");
  if (e && atoi(e) >= 32 && atoi(e) <= kSpmvTileRows) return atoi(e);
  int tr = kSpmvTileRows;
  while (tr > 128 && ceil_div(n, (int64_t)tr) < int64_t(sm_count()) * 4) tr /= 2;
  return tr;
}

static inline int spmv_blocks(int64_t n, int tile_rows) {
  const int64_t tiles = ceil_div(n, (int64_t)tile_rows);
  return (int)std::max<int64_t>(
      1, std::min<int64_t>(tiles, std::min<int64_t>(int64_t(sm_count()) * 8, kMaxVecBlocks)));
}

template <typename T>
static int spmv_launch(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                       const T* vals, const T* x, T* y, const double* norm2_parts, int n_parts,
                       double* beta_out, double* dot_parts, int* blocks_out, cudaStream_t st) {
  const char* form = getenv("GSPB200_SPMV");
  if (!(form && strcmp(form, "window") == 0)) {
    const int lpr = spmv_lanes_subwarp(n, nnz);
    const int64_t rpb = (kVecThreads / lpr) * 4;
    const int blocks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(n, rpb),
        std::min<int64_t>(int64_t(sm_count()) * 8, kMaxVecBlocks)));
    if (blocks_out) *blocks_out = blocks;
#define GSP_SPMV_SW(L)                                                                       \
  spmv_subwarp_kernel<T, L><<<blocks, kVecThreads, 0, st>>>(n, indptr, indices, vals, x, y, \
                                                             norm2_parts, n_parts, beta_out, \
                                                             dot_parts)
    switch (lpr) {
      case 2: GSP_SPMV_SW(2); break;
      case 4: GSP_SPMV_SW(4); break;
      case 8: GSP_SPMV_SW(8); break;
      case 16: GSP_SPMV_SW(16); break;
      default: GSP_SPMV_SW(32); break;
    }
#undef GSP_SPMV_SW
    GSP_LAUNCH_CHECK("spmv_subwarp");
    return GSP_OK;
  }
  const int lpr = spmv_lanes(n, nnz);
  const int tr = spmv_tile_rows(n);
  const int blocks = spmv_blocks(n, tr);
  if (blocks_out) *blocks_out = blocks;
#define GSP_SPMV(L)                                                                         \
  spmv_window_kernel<T, L><<<blocks, kVecThreads, 0, st>>>(n, indptr, indices, vals, x, y, \
                                                            norm2_parts, n_parts, beta_out, \
                                                            dot_parts, tr)
  switch (lpr) {
    case 2: GSP_SPMV(2); break;
    case 4: GSP_SPMV(4); break;
    case 8: GSP_SPMV(8); break;
    case 16: GSP_SPMV(16); break;
    default: GSP_SPMV(32); break;
  }
#undef GSP_SPMV
  GSP_LAUNCH_CHECK("spmv_window");
  return GSP_OK;
}

// ---------------------------------------------------------------- Lanczos
// The recurrence is carried on UNNORMALISED vectors u_j (v_j = u_j / beta_{j-1}), so that an
// iteration is two launches and no pass exists only to rescale a vector:
//   spmv   : beta_{j-1} = |u_j| from the partials of the previous update; w = L v_j;
//            partial sums of alpha_j = v_j' w                       (reads CSR + u_j, writes w)
//   update : alpha_j = sum(partials); u_{j+1} = w - alpha_j v_j - beta_{j-1} v_{j-1};
//            partial sums of |u_{j+1}|^2                            (3 reads, 1 write)
template <typename T>
__global__ void lanczos_update_kernel(int64_t n, T* __restrict__ w, const T* __restrict__ u,
                                      const T* __restrict__ u_prev, const double* dot_parts,
                                      int n_dot, const double* beta_j1, const double* beta_j2,
                                      double* alpha_out, double* norm2_parts) {
  const double a = sum_partials(dot_parts, n_dot);
  if (blockIdx.x == 0 && threadIdx.x == 0) *alpha_out = a;
  const double b1 = *beta_j1;                                  // |u_j|
  const double ca = b1 > 0 ? a / b1 : 0.0;                     // alpha_j v_j = (alpha_j / b1) u_j
  double cb = 0.0;                                             // beta_{j-1} v_{j-1} = (b1 / b2) u_{j-1}
  if (u_prev) {
    const double b2 = *beta_j2;
    cb = b2 > 0 ? b1 / b2 : 0.0;
  }
  double acc = 0;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    double t = double(w[i]) - ca * double(u[i]);
    if (u_prev) t -= cb * double(u_prev[i]);
    const T ts = T(t);
    w[i] = ts;
    acc += double(ts) * double(ts);
  }
  acc = block_allreduce(acc);
  if (threadIdx.x == 0) norm2_parts[blockIdx.x] = acc;
}

// beta_{j1-1} of the last iteration of a batch (the next spmv would compute it)
__global__ void lanczos_finish_kernel(const double* norm2_parts, int n_parts, double* beta_out) {
  const double nb = sqrt(sum_partials(norm2_parts, n_parts));
  if (threadIdx.x == 0) *beta_out = nb;
}

static inline int vec_blocks(int64_t n) {
  return (int)std::min<int64_t>(ceil_div(n > 0 ? n : 1, kVecThreads),
                                std::min<int64_t>(int64_t(sm_count()) * 8, kMaxVecBlocks));
}

// Iterations [j0, j1) of the recurrence.  V holds three n-vectors; u_j lives in slot j % 3.
// scal = alpha[0..cap) | beta[-1..cap) (cap + 1 values, beta[-1] = |u_0|) | partials A[2048]
//        | partials B[2048] | (n_a, n_b as doubles).
template <typename T>
int lanczos_run(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                const T* data, T* V, int j0, int j1, int cap, uint64_t seed, double* scal,
                cudaStream_t st) {
  GSP_REQUIRE(n >= 1 && j0 >= 0 && j1 <= cap && j0 <= j1, "bad Lanczos range");
  double* alpha = scal;
  double* beta = scal + cap + 1;                 // beta[-1] is valid
  double* part_a = scal + 2 * cap + 1;
  double* part_b = part_a + kMaxVecBlocks;
  const int gb = vec_blocks(n);
  if (j0 == 0) {
    GSP_CUDA(cudaMemsetAsync(scal, 0, sizeof(double) * (2 * cap + 1 + 2 * kMaxVecBlocks), st));
    lanczos_seed_kernel<T><<<gb, kVecThreads, 0, st>>>(n, V, seed, part_b);
    GSP_LAUNCH_CHECK("lanczos_seed");
  }
  for (int j = j0; j < j1; ++j) {
    T* u = V + int64_t(j % 3) * n;
    T* w = V + int64_t((j + 1) % 3) * n;
    const T* up = j > 0 ? V + int64_t((j + 2) % 3) * n : nullptr;
    int sb = 0;
    // w = L u_j / |u_j|, beta[j-1] = |u_j|, partials of alpha_j
    int rc = spmv_launch<T>(n, nnz, indptr, indices, data, u, w, part_b, gb, beta + j - 1, part_a,
                            &sb, st);
    if (rc != GSP_OK) return rc;
    lanczos_update_kernel<T><<<gb, kVecThreads, 0, st>>>(n, w, u, up, part_a, sb, beta + j - 1,
                                                         j > 0 ? beta + j - 2 : nullptr,
                                                         alpha + j, part_b);
    GSP_LAUNCH_CHECK("lanczos_update");
  }
  if (j1 > j0) {
    lanczos_finish_kernel<<<1, kVecThreads, 0, st>>>(part_b, gb, beta + j1 - 1);
    GSP_LAUNCH_CHECK("lanczos_finish");
  }
  return GSP_OK;
}

}  // namespace gsp

extern "C" {
int gsp_lanczos_f32(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                    const float* data, float* V3, int j0, int j1, int cap, uint64_t seed,
                    double* scal_dev, void* stream) {
  return gsp::lanczos_run<float>(n, nnz, indptr, indices, data, V3, j0, j1, cap, seed, scal_dev,
                                 gsp::as_stream(stream));
}
int gsp_lanczos_f64(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                    const double* data, double* V3, int j0, int j1, int cap, uint64_t seed,
                    double* scal_dev, void* stream) {
  return gsp::lanczos_run<double>(n, nnz, indptr, indices, data, V3, j0, j1, cap, seed, scal_dev,
                                  gsp::as_stream(stream));
}
// y = A x for one vector: scipy's csr_matvec (graph.py:911-917 through ARPACK, graph.py:955)
int gsp_spmv_f32(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                 const float* data, const float* x, float* y, void* stream) {
  if (n <= 0) return GSP_OK;
  return gsp::spmv_launch<float>(n, nnz, indptr, indices, data, x, y, nullptr, 0, nullptr, nullptr,
                                 nullptr, gsp::as_stream(stream));
}
int gsp_spmv_f64(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                 const double* data, const double* x, double* y, void* stream) {
  if (n <= 0) return GSP_OK;
  return gsp::spmv_launch<double>(n, nnz, indptr, indices, data, x, y, nullptr, 0, nullptr,
                                  nullptr, nullptr, gsp::as_stream(stream));
}
}
