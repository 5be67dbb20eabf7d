// Graph features of pygsp/features.py without the frame (pygsp_b200/features.py).
//
// Replaces, for pygsp/features.py and pygsp/filters/filter.py:
//   * s = np.identity(N) of compute_frame (filter.py:599), b columns at a time -> gsp_probe_block_*
//   * the row norms of the frame, np.linalg.norm(tig, axis=1) of compute_norm_tig
//     (features.py:58-59), through the diagonal Chebyshev moments
//     mu_n(i) = (T_n(Lt))_ii of the probe columns                -> gsp_cheby_moments_step_*,
//                                                                   gsp_cheby_moments_finish
//   * np.dot(G.A, G.A) of compute_avg_adj_deg (features.py:23) with G.A = W > 0
//     (graph.py:718-727)                                          -> gsp_two_hop_count_*
//
// The probe blocks T_k e_i themselves come from gsp_cheby_step_* (csrc/cheby.cu,
// csrc/cheby_tiled.cu), driven by filters/approximations.py:cheby_moments_device.
//
// Moments.  With T_j T_k = (T_{j+k} + T_{|j-k|}) / 2 and L symmetric,
//   mu_{2k} = 2 ||T_k e_i||^2 - 1,  mu_{2k+1} = 2 <T_{k+1} e_i, T_k e_i> - mu_1,  mu_1 = <T_1 e_i, e_i>.
// After step k (T_{k+1} from T_k) one pass sums ||T_{k+1}[:, j]||^2 and <T_{k+1}[:, j], T_k[:, j]>
// per column, in double also for float blocks, by the two-level column reduction of
// csrc/reduce.cuh, so a vertex's moments do not depend on the block width, its position in the
// block or the other vertices of the block.
//
// Two-hop counts.  For every row i, the number of distinct c with W[i, k] > 0 and W[k, c] > 0
// for some k (the entries of row i of the boolean product A A) and the number of k with
// W[i, k] > 0.  A row's candidates number cand_i = sum over its neighbours k of deg(k).  Rows
// with cand_i <= kLightCap are counted by one warp in a shared-memory hash set; heavier rows by
// a hash set of 2 cand_i slots (rounded up to a power of two) in global memory, the heavy rows
// processed in chunks whose tables hold at most kHeavySlots slots together (a single row may
// exceed it: its table is at most 2 nnz slots, since cand_i <= nnz).  Counting successful
// insertions gives the same integer whatever the insertion order.
#include <vector>

#include "reduce.cuh"

namespace gsp {
namespace {

constexpr int kLightCap = 1024;               // candidates of a row counted in shared memory
constexpr int kLightSlots = 2 * kLightCap;    // hash slots per warp
constexpr int kLightWarps = 4;                // warps per CTA of the light-row kernel (32 KB)
constexpr int64_t kHeavySlots = int64_t(1) << 24;   // global hash slots per heavy chunk (64 MB)
constexpr int kHeavySlices = 32;              // CTAs per heavy row

// X[r, j] = (r == v0 + j): columns v0 .. v0 + b - 1 of the identity, row-major (n, b)
template <typename T>
__global__ void probe_block_kernel(int64_t n, int64_t v0, int64_t b, T* __restrict__ X) {
  const int64_t count = n * b;
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < count;
       e += int64_t(gridDim.x) * blockDim.x) {
    const int64_t r = e / b, j = e - r * b;
    X[e] = r == v0 + j ? T(1) : T(0);
  }
}

// part[p][0][j] = partial sum of tn[r, j]^2, part[p][1][j] = partial sum of tn[r, j] tc[r, j],
// each in the order of column_part (csrc/reduce.cuh)
template <typename T>
__global__ void __launch_bounds__(kThreads)
moments_part_kernel(int64_t n, const T* __restrict__ tn, const T* __restrict__ tc, int64_t b,
                    int64_t chunk, double* __restrict__ part) {
  __shared__ double sums[2][kWarps][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t j = int64_t(blockIdx.y) * 32 + lane;
  const int64_t rb = int64_t(blockIdx.x) * chunk, re = min(n, rb + chunk);
  double sq = 0.0, cr = 0.0;
  if (j < b) {
#pragma unroll 4
    for (int64_t r = rb + w; r < re; r += kWarps) {
      const double a = double(__ldcs(tn + r * b + j)), c = double(__ldcs(tc + r * b + j));
      sq = fma(a, a, sq);
      cr = fma(a, c, cr);
    }
  }
  sums[0][w][lane] = sq;
  sums[1][w][lane] = cr;
  __syncthreads();
  if (w == 0 && j < b) {
    double s0 = 0.0, s1 = 0.0;
    for (int q = 0; q < kWarps; ++q) {
      s0 += sums[0][q][lane];
      s1 += sums[1][q][lane];
    }
    double* out = part + int64_t(blockIdx.x) * 2 * b;
    out[j] = s0;
    out[b + j] = s1;
  }
}

// mu[v0 + j, :] from sums (m, 2, b): sums[k][0] = ||T_{k+1}||^2, sums[k][1] = <T_{k+1}, T_k>
__global__ void moments_finish_kernel(int m, int64_t v0, int64_t b,
                                      const double* __restrict__ sums, double* __restrict__ mu) {
  const int64_t j = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (j >= b) return;
  const int64_t width = 2 * int64_t(m) + 1;
  double* row = mu + (v0 + j) * width;
  const double mu1 = sums[b + j];
  row[0] = 1.0;
  row[1] = mu1;
  for (int k = 1; k <= m; ++k) {
    row[2 * k] = 2.0 * sums[(int64_t(k - 1) * 2) * b + j] - 1.0;
    if (k < m) row[2 * k + 1] = 2.0 * sums[(int64_t(k) * 2 + 1) * b + j] - mu1;
  }
}

// --------------------------------------------------------------------- two-hop counts
__device__ __forceinline__ uint32_t slot_hash(int32_t c) { return uint32_t(c) * 2654435761u; }

// deg[i] = #{e in row i : data[e] > 0}
template <typename T>
__global__ void two_hop_degree_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                      const T* __restrict__ data, int32_t* __restrict__ deg) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    int32_t d = 0;
    for (int32_t e = indptr[i]; e < indptr[i + 1]; ++e) d += data[e] > T(0);
    deg[i] = d;
  }
}

// cand[i] = sum_{e in row i, data[e] > 0} deg[indices[e]]; one warp per row
template <typename T>
__global__ void two_hop_cand_kernel(int64_t n, const int32_t* __restrict__ indptr,
                                    const int32_t* __restrict__ indices, const T* __restrict__ data,
                                    const int32_t* __restrict__ deg, int64_t* __restrict__ cand) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = int64_t(gridDim.x) * (blockDim.x >> 5);
  for (int64_t i = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; i < n; i += warps) {
    int64_t s = 0;
    for (int32_t e = indptr[i] + lane; e < indptr[i + 1]; e += 32)
      if (data[e] > T(0)) s += deg[indices[e]];
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) cand[i] = s;
  }
}

// Rows with cand <= kLightCap: one warp, a hash set of 2 cand slots (a power of two, >= 32) in
// shared memory.  Heavier rows get two_hop = 0 and are counted by two_hop_heavy_kernel.
template <typename T>
__global__ void __launch_bounds__(kLightWarps * 32)
two_hop_light_kernel(int64_t n, const int32_t* __restrict__ indptr,
                     const int32_t* __restrict__ indices, const T* __restrict__ data,
                     const int64_t* __restrict__ cand, int32_t* __restrict__ two_hop) {
  __shared__ int32_t table[kLightWarps][kLightSlots];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int32_t* set = table[w];
  const int64_t warps = int64_t(gridDim.x) * kLightWarps;
  for (int64_t i = int64_t(blockIdx.x) * kLightWarps + w; i < n; i += warps) {
    const int64_t ci = cand[i];
    if (ci > kLightCap) {
      if (lane == 0) two_hop[i] = 0;
      continue;
    }
    int size = 32;
    while (size < 2 * ci) size <<= 1;
    const uint32_t mask = uint32_t(size - 1);
    for (int s = lane; s < size; s += 32) set[s] = -1;
    __syncwarp();
    int32_t count = 0;
    for (int32_t e = indptr[i]; e < indptr[i + 1]; ++e) {
      if (!(data[e] > T(0))) continue;
      const int32_t k = indices[e];
      const int32_t kb = indptr[k], ke = indptr[k + 1];
      for (int32_t f0 = kb; f0 < ke; f0 += 32) {
        const int32_t f = f0 + lane;
        bool fresh = false;
        if (f < ke && data[f] > T(0)) {
          const int32_t c = indices[f];
          uint32_t h = slot_hash(c) & mask;
          while (true) {
            const int32_t prev = atomicCAS(&set[h], -1, c);
            if (prev == -1) { fresh = true; break; }
            if (prev == c) break;
            h = (h + 1) & mask;
          }
        }
        count += __popc(__ballot_sync(0xffffffffu, fresh));
      }
    }
    if (lane == 0) two_hop[i] = count;
    __syncwarp();
  }
}

// One heavy row per blockIdx.y (rows[y], its table at table + offs[y] with size[y] slots, a
// power of two, filled with -1).  Warp (blockIdx.x, w) takes the row's neighbour entries
// x * 8 + w, stepping by gridDim.x * 8; its lanes stride the neighbour's row.
template <typename T>
__global__ void __launch_bounds__(kThreads)
two_hop_heavy_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                     const T* __restrict__ data, const int32_t* __restrict__ rows,
                     const int64_t* __restrict__ offs, const int64_t* __restrict__ sizes,
                     int32_t* __restrict__ table, int32_t* __restrict__ two_hop) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int32_t i = rows[blockIdx.y];
  int32_t* set = table + offs[blockIdx.y];
  const uint64_t mask = uint64_t(sizes[blockIdx.y] - 1);
  const int32_t stride = int32_t(gridDim.x) * kWarps;
  int32_t count = 0;
  for (int32_t e = indptr[i] + int32_t(blockIdx.x) * kWarps + w; e < indptr[i + 1]; e += stride) {
    if (!(data[e] > T(0))) continue;
    const int32_t k = indices[e];
    const int32_t kb = indptr[k], ke = indptr[k + 1];
    for (int32_t f0 = kb; f0 < ke; f0 += 32) {
      const int32_t f = f0 + lane;
      bool fresh = false;
      if (f < ke && data[f] > T(0)) {
        const int32_t c = indices[f];
        uint64_t h = uint64_t(slot_hash(c)) & mask;
        while (true) {
          const int32_t prev = atomicCAS(&set[h], -1, c);
          if (prev == -1) { fresh = true; break; }
          if (prev == c) break;
          h = (h + 1) & mask;
        }
      }
      count += __popc(__ballot_sync(0xffffffffu, fresh));
    }
  }
  if (lane == 0 && count) atomicAdd(&two_hop[i], count);
}

// heavy row list: ids of the rows with cand > kLightCap (order fixed on the host afterwards)
__global__ void two_hop_select_kernel(int64_t n, const int64_t* __restrict__ cand,
                                      int32_t* __restrict__ ids, int64_t* __restrict__ ids_cand,
                                      unsigned long long* __restrict__ count) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    if (cand[i] > kLightCap) {
      const unsigned long long q = atomicAdd(count, 1ull);
      ids[q] = int32_t(i);
      ids_cand[q] = cand[i];
    }
  }
}

template <typename T>
int moments_step(int64_t n, const T* tn, const T* tc, int64_t b, int m, int k, double* sums,
                 cudaStream_t st) {
  GSP_REQUIRE(n >= 1 && b >= 1 && m >= 1 && k >= 0 && k < m, "bad sizes");
  GSP_REQUIRE(ceil_div(b, 32) < 65536, "block too wide");
  const Parts P = row_parts(n);
  Scratch<double> part(st);
  GSP_CUDA(part.alloc(P.used * 2 * b));
  moments_part_kernel<T><<<dim3((unsigned)P.used, (unsigned)ceil_div(b, 32)), kThreads, 0, st>>>(
      n, tn, tc, b, P.chunk, part.get());
  GSP_LAUNCH_CHECK("moments_part");
  return sum_parts(part.get(), P.used, 2 * b, sums + int64_t(k) * 2 * b, st);
}

template <typename T>
int two_hop_count(int64_t n, const int32_t* indptr, const int32_t* indices, const T* data,
                  int32_t* two_hop, int32_t* degree, cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31), "bad sizes");
  if (n == 0) return GSP_OK;
  // scratch: cand (n), heavy ids' candidate counts (n), heavy ids (n), counter
  Scratch<char> scratch(st);
  GSP_CUDA(scratch.alloc(size_t(n) * (8 + 8 + 4) + 8));
  int64_t* cand = reinterpret_cast<int64_t*>(scratch.get());
  int64_t* ids_cand = cand + n;
  unsigned long long* counter = reinterpret_cast<unsigned long long*>(ids_cand + n);
  int32_t* ids = reinterpret_cast<int32_t*>(counter + 1);
  two_hop_degree_kernel<T><<<grid_for(n), kThreads, 0, st>>>(n, indptr, data, degree);
  GSP_LAUNCH_CHECK("two_hop_degree");
  two_hop_cand_kernel<T><<<grid_for(n * 32), kThreads, 0, st>>>(n, indptr, indices, data, degree,
                                                                 cand);
  GSP_LAUNCH_CHECK("two_hop_cand");
  two_hop_light_kernel<T><<<(unsigned)std::min<int64_t>(ceil_div(n, kLightWarps), 65535),
                            kLightWarps * 32, 0, st>>>(n, indptr, indices, data, cand, two_hop);
  GSP_LAUNCH_CHECK("two_hop_light");
  GSP_CUDA(cudaMemsetAsync(counter, 0, 8, st));
  two_hop_select_kernel<<<grid_for(n), kThreads, 0, st>>>(n, cand, ids, ids_cand, counter);
  GSP_LAUNCH_CHECK("two_hop_select");
  unsigned long long heavy = 0;
  GSP_CUDA(cudaMemcpyAsync(&heavy, counter, 8, cudaMemcpyDeviceToHost, st));
  GSP_CUDA(cudaStreamSynchronize(st));
  if (heavy == 0) return GSP_OK;
  std::vector<int32_t> hid(heavy);
  std::vector<int64_t> hc(heavy);
  GSP_CUDA(cudaMemcpyAsync(hid.data(), ids, heavy * 4, cudaMemcpyDeviceToHost, st));
  GSP_CUDA(cudaMemcpyAsync(hc.data(), ids_cand, heavy * 8, cudaMemcpyDeviceToHost, st));
  GSP_CUDA(cudaStreamSynchronize(st));
  // process the heavy rows in increasing id order (the selection's order is not fixed)
  std::vector<size_t> order(heavy);
  for (size_t q = 0; q < heavy; ++q) order[q] = q;
  std::sort(order.begin(), order.end(), [&](size_t a, size_t c) { return hid[a] < hid[c]; });
  std::vector<int64_t> size(heavy);
  int64_t widest = 0;
  for (size_t q = 0; q < heavy; ++q) {
    int64_t s = 1;
    while (s < 2 * hc[q]) s <<= 1;
    size[q] = s;
    widest = std::max(widest, s);
  }
  const int64_t budget = std::max(kHeavySlots, widest);
  const int64_t max_rows = 65535;
  Scratch<int32_t> table(st);
  Scratch<int64_t> meta(st);
  GSP_CUDA(table.alloc(budget));
  GSP_CUDA(meta.alloc(max_rows * 3));
  int64_t* d_offs = meta.get();
  int64_t* d_sizes = d_offs + max_rows;
  int32_t* d_rows = reinterpret_cast<int32_t*>(d_offs + 2 * max_rows);
  std::vector<int32_t> rows;
  std::vector<int64_t> offs, sizes;
  for (size_t q0 = 0; q0 < heavy;) {
    rows.clear();
    offs.clear();
    sizes.clear();
    int64_t used = 0;
    size_t q = q0;
    for (; q < heavy && int64_t(rows.size()) < max_rows; ++q) {
      const size_t o = order[q];
      if (used + size[o] > budget) break;
      rows.push_back(hid[o]);
      offs.push_back(used);
      sizes.push_back(size[o]);
      used += size[o];
    }
    q0 = q;
    const size_t nr = rows.size();
    // the host vectors must outlive the copies: synchronise before the next chunk refills them
    GSP_CUDA(cudaMemsetAsync(table.get(), 0xFF, used * sizeof(int32_t), st));
    GSP_CUDA(cudaMemcpyAsync(d_rows, rows.data(), nr * 4, cudaMemcpyHostToDevice, st));
    GSP_CUDA(cudaMemcpyAsync(d_offs, offs.data(), nr * 8, cudaMemcpyHostToDevice, st));
    GSP_CUDA(cudaMemcpyAsync(d_sizes, sizes.data(), nr * 8, cudaMemcpyHostToDevice, st));
    two_hop_heavy_kernel<T><<<dim3(kHeavySlices, (unsigned)nr), kThreads, 0, st>>>(
        indptr, indices, data, d_rows, d_offs, d_sizes, table.get(), two_hop);
    GSP_LAUNCH_CHECK("two_hop_heavy");
    GSP_CUDA(cudaStreamSynchronize(st));
  }
  return GSP_OK;
}

}  // namespace
}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {

#define GSP_MOMENTS_API(SUF, T)                                                                    \
  int gsp_probe_block_##SUF(int64_t n, int64_t v0, int64_t b, T* X, void* stream) {                \
    GSP_REQUIRE(n >= 1 && b >= 1 && v0 >= 0 && v0 + b <= n, "bad sizes");                         \
    gsp::probe_block_kernel<T><<<gsp::grid_for(n * b), gsp::kThreads, 0, gsp::as_stream(stream)>>>( \
        n, v0, b, X);                                                                              \
    GSP_LAUNCH_CHECK("probe_block");                                                               \
    return GSP_OK;                                                                                 \
  }                                                                                                \
  int gsp_cheby_moments_step_##SUF(int64_t n, const T* t_next, const T* t_cur, int64_t b, int m,  \
                                   int k, double* sums, void* stream) {                            \
    return gsp::moments_step<T>(n, t_next, t_cur, b, m, k, sums, gsp::as_stream(stream));          \
  }                                                                                                \
  int gsp_two_hop_count_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices,           \
                              const T* data, int32_t* two_hop, int32_t* degree, void* stream) {    \
    return gsp::two_hop_count<T>(n, indptr, indices, data, two_hop, degree,                        \
                                 gsp::as_stream(stream));                                          \
  }

GSP_MOMENTS_API(f32, float)
GSP_MOMENTS_API(f64, double)

int gsp_cheby_moments_finish(int64_t n, int m, int64_t v0, int64_t b, const double* sums,
                             double* mu, void* stream) {
  GSP_REQUIRE(n >= 1 && m >= 1 && b >= 1 && v0 >= 0 && v0 + b <= n, "bad sizes");
  gsp::moments_finish_kernel<<<gsp::grid_for(b), gsp::kThreads, 0, gsp::as_stream(stream)>>>(
      m, v0, b, sums, mu);
  GSP_LAUNCH_CHECK("moments_finish");
  return GSP_OK;
}

}  // extern "C"
