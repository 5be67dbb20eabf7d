// Random graph models (pygsp/graphs/stochasticblockmodel.py, erdosrenyi.py, barabasialbert.py):
// the stochastic block model's pair sampler and Barabasi-Albert preferential attachment.
//
// Replaces:
//   * the N^2 loop of one uniform per vertex pair of stochasticblockmodel.py:125-139 (and so of
//     ErdosRenyi, its k = 1 case)                         -> gsp_sbm_count + gsp_sbm_fill
//   * the per-vertex W.sum / rng.choice(replace=False, p) loop of barabasialbert.py:54-64
//                                                         -> gsp_barabasi_albert
//
// Every draw comes from a counter-based Philox4x32-10 stream of curand_kernel.h, keyed by the
// caller's 64-bit key, whose subsequence is a chunk id (SBM) or a slot id (BA).  A result is a
// function of the key and the parameters only: grid size, block size and, for BA, the number
// of rounds do not enter it, so a serial restatement of either sampler gives the same graph.
//
// SBM.  Block pair b's candidate pairs are the index range [0, n_b), cut by the caller into
// chunks of clen_b indices (the last one shorter); chunks are numbered globally from cfirst_b.
// A chunk walks the Bernoulli(p_b) process over its range by geometric skips: from position
// pos, the next success is pos + 1 + floor(log(u) / log1p(-p_b)), u in (0, 1] built from 53
// random bits, the chunk's uniforms taken in order, two per curand4.  p_b = 1 takes every index
// without drawing.  The count pass writes the number of COO entries each chunk emits and scans
// them into offsets; the fill pass regenerates the same walk (the same function, FILL = true)
// and writes the entries there.  An index decodes into block-local (i, j) by the block's kind:
//   kRect       i = idx / nb, j = idx % nb                     (off-diagonal, or directed with loops)
//   kTriStrict  i > j, idx = i (i - 1) / 2 + j                  (undirected, no loops)
//   kTriLoops   i >= j, idx = i (i + 1) / 2 + j                 (undirected with loops)
//   kOffDiag    i = idx / (n - 1), j = idx % (n - 1) skipping i (directed, no loops)
// The square roots are corrected in integers, so every decoder is a bijection.  Local ids map to
// vertices through perm (the stable sort of z).  An undirected off-diagonal pair emits both
// orientations, a loop once.
//
// BA.  Slot (i, s), i in [m0, N), s < m, has id (i - m0) m + s.  Attempt k of a slot draws one
// 64-bit uniform (stream `slot`, offset 4k) and r = mulhi(u, W_i), W_i = i + 2 m (i - m0), the
// total weight sum_{j<i} (1 + deg_j) of barabasialbert.py:55-56.  r < i picks vertex r; else
// q = r - i is a position in the list of edge endpoints: edge e = q / 2 was made by slot e, of
// vertex m0 + e / m, which is its even endpoint; the odd one is slot e's final target.  A slot
// is final once its value is known and differs from the vertex's earlier slots; a duplicate
// redraws with attempt k + 1, which is successive sampling, the law of choice(replace=False, p).
// One round is one launch over the vertices: each walks its slots in order, takes a pointee's
// value once that pointee is final (a final value never changes: no ordering beyond a single
// 32-bit volatile load is needed) and stops at a pointee that is not, until the next round.
// No thread waits for another.  The lowest non-final slot always finalises, so the rounds end;
// the host reads the pending count every kCheckEvery rounds and gives up after kMaxRounds.
#include <cub/cub.cuh>
#include <curand_kernel.h>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {
namespace {

constexpr int kThreads = 256;
constexpr int kRect = 0, kTriStrict = 1, kTriLoops = 2;   // 3: n (n - 1) ordered pairs
constexpr int kPlanCols = GSPB200_SBM_PLAN_COLS;
constexpr int kCheckEvery = 4;
constexpr int kMaxRounds = 4096;

__device__ __forceinline__ double unit53(unsigned long long r) {
  return double((r >> 11) + 1) * 0x1.0p-53;         // (0, 1]
}

// block-local (i, j) of candidate index idx
__device__ __forceinline__ void decode(int kind, int64_t idx, int64_t nb, int64_t& i,
                                       int64_t& j) {
  if (kind == kRect) {
    i = idx / nb;
    j = idx - i * nb;
  } else if (kind == kTriStrict) {
    i = (int64_t)floor((1.0 + sqrt(1.0 + 8.0 * double(idx))) * 0.5);
    while (i * (i - 1) / 2 > idx) --i;
    while ((i + 1) * i / 2 <= idx) ++i;
    j = idx - i * (i - 1) / 2;
  } else if (kind == kTriLoops) {
    i = (int64_t)floor((sqrt(1.0 + 8.0 * double(idx)) - 1.0) * 0.5);
    while (i * (i + 1) / 2 > idx) --i;
    while ((i + 1) * (i + 2) / 2 <= idx) ++i;
    j = idx - i * (i + 1) / 2;
  } else {                                            // kOffDiag, nb = n
    i = idx / (nb - 1);
    j = idx - i * (nb - 1);
    j += (j >= i);
  }
}

// Walks chunk c.  COUNT: returns the entries it emits.  FILL: also writes them from out.
template <bool FILL>
__device__ int64_t walk_chunk(int64_t c, int64_t nblk, const int64_t* __restrict__ plan,
                              const double* __restrict__ prob, uint64_t key,
                              const int32_t* __restrict__ perm, int32_t* rows, int32_t* cols,
                              int64_t out) {
  int lo = 0, hi = (int)nblk - 1;                     // last block pair with cfirst <= c
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(plan + mid * kPlanCols + 2) <= c) lo = mid; else hi = mid - 1;
  }
  const int64_t* row = plan + lo * kPlanCols;
  const int64_t n_pairs = __ldg(row + 0), clen = __ldg(row + 1), cfirst = __ldg(row + 2);
  const int64_t row0 = __ldg(row + 3), col0 = __ldg(row + 4), nb = __ldg(row + 5);
  const int kind = (int)__ldg(row + 6);
  const bool mirror = __ldg(row + 7) != 0;
  const double p = __ldg(prob + 2 * lo), lq = __ldg(prob + 2 * lo + 1);
  const int64_t idx0 = (c - cfirst) * clen;
  const int64_t idx1 = idx0 + clen < n_pairs ? idx0 + clen : n_pairs;

  curandStatePhilox4_32_10_t state;
  const bool every = p >= 1.0;
  if (!every) curand_init(key, (unsigned long long)c, 0ull, &state);
  uint4 r4 = make_uint4(0, 0, 0, 0);
  bool second = false;
  int64_t emitted = 0, pos = idx0 - 1;
  while (true) {
    if (every) {
      ++pos;
    } else {
      unsigned long long r;
      if (!second) {
        r4 = curand4(&state);
        r = (uint64_t(r4.x) << 32) | r4.y;
      } else {
        r = (uint64_t(r4.z) << 32) | r4.w;
      }
      second = !second;
      const double skip = floor(log(unit53(r)) / lq);
      if (skip >= double(idx1 - pos - 1)) break;      // compared in double: no overflow
      pos += 1 + (int64_t)skip;
    }
    if (pos >= idx1) break;
    int64_t i, j;
    decode(kind, pos, nb, i, j);
    const bool both = mirror && !(kind != kRect && i == j);
    if (FILL) {
      const int32_t u = __ldg(perm + row0 + i), v = __ldg(perm + col0 + j);
      rows[out + emitted] = u;
      cols[out + emitted] = v;
      if (both) {
        rows[out + emitted + 1] = v;
        cols[out + emitted + 1] = u;
      }
    }
    emitted += both ? 2 : 1;
  }
  return emitted;
}

__global__ void __launch_bounds__(kThreads)
sbm_count_kernel(int64_t n_chunks, int64_t nblk, const int64_t* __restrict__ plan,
                 const double* __restrict__ prob, uint64_t key, int64_t* counts) {
  for (int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; c < n_chunks;
       c += int64_t(gridDim.x) * blockDim.x)
    counts[c] = walk_chunk<false>(c, nblk, plan, prob, key, nullptr, nullptr, nullptr, 0);
}

__global__ void __launch_bounds__(kThreads)
sbm_fill_kernel(int64_t n_chunks, int64_t nblk, const int64_t* __restrict__ plan,
                const double* __restrict__ prob, uint64_t key, const int32_t* __restrict__ perm,
                const int64_t* __restrict__ offsets, int32_t* rows, int32_t* cols) {
  for (int64_t c = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; c < n_chunks;
       c += int64_t(gridDim.x) * blockDim.x)
    walk_chunk<true>(c, nblk, plan, prob, key, perm, rows, cols, __ldg(offsets + c));
}

// One round over the vertices (see the file comment).  target: final value per slot, -1 while
// not final; done / attempt: per vertex, its number of final slots and the attempt of the first
// slot that is not.
__global__ void __launch_bounds__(kThreads)
ba_round_kernel(int64_t n, int64_t m0, int64_t m, uint64_t key, int32_t* target,
                int32_t* done, int32_t* attempt, unsigned long long* pending) {
  volatile int32_t* vt = target;
  int open = 0;
  for (int64_t i = m0 + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    int64_t s = done[i];
    if (s == m) continue;
    int k = attempt[i];
    const int64_t base = (i - m0) * m;
    const unsigned long long w = (unsigned long long)(i + 2 * m * (i - m0));
    while (s < m) {
      curandStatePhilox4_32_10_t state;
      curand_init(key, (unsigned long long)(base + s), 4ull * (unsigned)k, &state);
      const uint4 r4 = curand4(&state);
      const unsigned long long r = __umul64hi((uint64_t(r4.x) << 32) | r4.y, w);
      int32_t v;
      if (r < (unsigned long long)i) {
        v = (int32_t)r;
      } else {
        const unsigned long long q = r - (unsigned long long)i;
        if ((q & 1) == 0) {
          v = (int32_t)(m0 + (int64_t)(q >> 1) / m);
        } else {
          v = vt[q >> 1];
          if (v < 0) break;                           // pointee not final yet: next round
        }
      }
      bool dup = false;
      for (int64_t t = 0; t < s; ++t) dup |= vt[base + t] == v;
      if (dup) {
        ++k;
        continue;
      }
      vt[base + s] = v;
      ++s;
      k = 0;
    }
    done[i] = (int32_t)s;
    attempt[i] = k;
    open += s < m;
  }
  const int block_open = __syncthreads_count(open);
  if (threadIdx.x == 0 && block_open) atomicAdd(pending, (unsigned long long)block_open);
}

__global__ void ba_emit_kernel(int64_t slots, int64_t m0, int64_t m,
                               const int32_t* __restrict__ target, int32_t* rows, int32_t* cols) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= slots) return;
  const int32_t i = (int32_t)(m0 + e / m), v = __ldg(target + e);
  rows[2 * e] = i;
  cols[2 * e] = v;
  rows[2 * e + 1] = v;
  cols[2 * e + 1] = i;
}

int grid_of(int64_t work, int max_blocks) {
  int64_t g = ceil_div(work, kThreads);
  if (max_blocks > 0 && g > max_blocks) g = max_blocks;
  const int64_t cap = int64_t(sm_count()) * 32;
  return (int)std::max<int64_t>(1, std::min(g, cap));
}

}  // namespace

int sbm_count(int64_t n_chunks, int64_t nblk, const int64_t* plan, const double* prob,
              uint64_t key, int64_t* offsets, int max_blocks, cudaStream_t st) {
  GSP_CUDA(cudaMemsetAsync(offsets, 0, sizeof(int64_t), st));
  if (n_chunks == 0) return GSP_OK;
  sbm_count_kernel<<<grid_of(n_chunks, max_blocks), kThreads, 0, st>>>(n_chunks, nblk, plan,
                                                                      prob, key, offsets + 1);
  GSP_LAUNCH_CHECK("sbm_count");
  return cub_temp("cub::DeviceScan::InclusiveSum", st, [&](void* tmp, size_t& bytes) {
    return cub::DeviceScan::InclusiveSum(tmp, bytes, offsets + 1, offsets + 1, n_chunks, st);
  });
}

int sbm_fill(int64_t n_chunks, int64_t nblk, const int64_t* plan, const double* prob,
             uint64_t key, const int32_t* perm, const int64_t* offsets, int32_t* rows,
             int32_t* cols, int max_blocks, cudaStream_t st) {
  if (n_chunks == 0) return GSP_OK;
  sbm_fill_kernel<<<grid_of(n_chunks, max_blocks), kThreads, 0, st>>>(
      n_chunks, nblk, plan, prob, key, perm, offsets, rows, cols);
  GSP_LAUNCH_CHECK("sbm_fill");
  return GSP_OK;
}

int barabasi_albert(int64_t n, int64_t m0, int64_t m, uint64_t key, int32_t* rows, int32_t* cols,
                    int max_blocks, int* rounds, cudaStream_t st) {
  *rounds = 0;
  if (n <= m0) return GSP_OK;
  const int64_t slots = m * (n - m0);
  Scratch<int32_t> target(st), state(st);
  Scratch<unsigned long long> pending(st);
  GSP_CUDA(target.alloc(slots));
  GSP_CUDA(state.alloc(2 * n));
  GSP_CUDA(pending.alloc(1));
  GSP_CUDA(cudaMemsetAsync(target.get(), 0xff, sizeof(int32_t) * slots, st));
  GSP_CUDA(cudaMemsetAsync(state.get(), 0, sizeof(int32_t) * 2 * n, st));
  int32_t* done = state.get();
  int32_t* attempt = state.get() + n;
  const int grid = grid_of(n - m0, max_blocks);
  unsigned long long open = 1;
  int r = 0;
  while (open != 0) {
    if (r == kMaxRounds)
      return fail(GSP_ERR_UNSUPPORTED, "barabasi_albert: slots still open after %s rounds",
                  "4096");
    GSP_CUDA(cudaMemsetAsync(pending.get(), 0, sizeof(unsigned long long), st));
    ba_round_kernel<<<grid, kThreads, 0, st>>>(n, m0, m, key, target.get(), done, attempt,
                                               pending.get());
    GSP_LAUNCH_CHECK("ba_round");
    ++r;
    if (r % kCheckEvery == 0) {
      GSP_CUDA(cudaMemcpyAsync(&open, pending.get(), sizeof(open), cudaMemcpyDeviceToHost, st));
      GSP_CUDA(cudaStreamSynchronize(st));
    }
  }
  *rounds = r;
  ba_emit_kernel<<<(unsigned)ceil_div(slots, kThreads), kThreads, 0, st>>>(slots, m0, m,
                                                                        target.get(), rows, cols);
  GSP_LAUNCH_CHECK("ba_emit");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {
int gsp_sbm_count(int64_t n_chunks, int64_t n_blocks, const int64_t* plan, const double* prob,
                  uint64_t key, int64_t* offsets, int max_blocks, void* stream) {
  GSP_REQUIRE(n_chunks >= 0 && n_blocks >= 0 && n_blocks < (int64_t(1) << 31) && offsets,
              "bad arguments");
  GSP_REQUIRE(n_chunks == 0 || (n_blocks > 0 && plan && prob), "empty plan");
  return gsp::sbm_count(n_chunks, n_blocks, plan, prob, key, offsets, max_blocks,
                        gsp::as_stream(stream));
}
int gsp_sbm_fill(int64_t n_chunks, int64_t n_blocks, const int64_t* plan, const double* prob,
                 uint64_t key, const int32_t* perm, const int64_t* offsets, int32_t* rows,
                 int32_t* cols, int max_blocks, void* stream) {
  GSP_REQUIRE(n_chunks >= 0 && n_blocks >= 0 && n_blocks < (int64_t(1) << 31), "bad arguments");
  GSP_REQUIRE(n_chunks == 0 || (n_blocks > 0 && plan && prob && perm && offsets),
              "empty plan");
  return gsp::sbm_fill(n_chunks, n_blocks, plan, prob, key, perm, offsets, rows, cols,
                       max_blocks, gsp::as_stream(stream));
}
int gsp_barabasi_albert(int64_t n, int64_t m0, int64_t m, uint64_t key, int32_t* rows,
                        int32_t* cols, int max_blocks, int* rounds_host_out, void* stream) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31) && m >= 1 && m0 >= m && rounds_host_out,
              "bad arguments");
  GSP_REQUIRE(n <= m0 || 2 * m * (n - m0) < (int64_t(1) << 31), "too many edges");
  return gsp::barabasi_albert(n, m0, m, key, rows, cols, max_blocks, rounds_host_out,
                              gsp::as_stream(stream));
}
}
