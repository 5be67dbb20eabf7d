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
//
// Exact-size subsets.  gsp_subset_select keeps a uniform n_s-subset of the candidate pairs the
// SBM walk drew for each pair space s (a run of consecutive plan rows, walked with no mirror at
// an inflated probability; the caller redraws when a space came up short).  Each candidate
// (u, v) gets the 64-bit priority of the first two words of the Philox block (g, 2^63) of the
// caller's key, g = u n + v its global pair index: one radix sort by priority, one stable radix
// sort by space, and the first n_s of each space are kept, both orientations emitted.  Given
// the walk's count k >= n_s, the walk's set is a uniform k-subset and the n_s lowest of k iid
// priorities a uniform n_s-subset of it.  Ties (equal priorities) go to the earlier candidate.
#include <cub/cub.cuh>
#include <curand_kernel.h>

#include <vector>

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

// position of x among the n + 1 non-decreasing offsets: the last s < n with off[s] <= x
__device__ __forceinline__ int64_t segment_of(const int64_t* __restrict__ off, int64_t n,
                                              int64_t x) {
  int64_t lo = 0, hi = n - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (__ldg(off + mid) <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void subset_begin_kernel(int64_t n_spaces, const int64_t* __restrict__ space_chunk,
                                    const int64_t* __restrict__ offsets, int64_t* begin) {
  const int64_t s = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (s <= n_spaces) begin[s] = __ldg(offsets + __ldg(space_chunk + s));
}

__global__ void __launch_bounds__(kThreads)
subset_priority_kernel(int64_t n_cand, int64_t n, const int32_t* __restrict__ rows,
                       const int32_t* __restrict__ cols, uint64_t key,
                       unsigned long long* prio, int32_t* pos) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < n_cand;
       e += int64_t(gridDim.x) * blockDim.x) {
    const uint64_t g = uint64_t(__ldg(rows + e)) * uint64_t(n) + uint64_t(__ldg(cols + e));
    curandStatePhilox4_32_10_t state;
    curand_init(key, 1ull << 63, 4ull * g, &state);
    const uint4 r4 = curand4(&state);
    prio[e] = (uint64_t(r4.x) << 32) | r4.y;
    pos[e] = (int32_t)e;
  }
}

__global__ void __launch_bounds__(kThreads)
subset_space_kernel(int64_t n_cand, int64_t n_spaces, const int64_t* __restrict__ begin,
                    const int32_t* __restrict__ pos, int32_t* space) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < n_cand;
       e += int64_t(gridDim.x) * blockDim.x)
    space[e] = (int32_t)segment_of(begin, n_spaces, __ldg(pos + e));
}

// output pair o of space s is the (o - sel[s])-th candidate of s in (priority, position) order
__global__ void __launch_bounds__(kThreads)
subset_emit_kernel(int64_t total, int64_t n_spaces, const int64_t* __restrict__ sel,
                   const int64_t* __restrict__ begin, const int32_t* __restrict__ order,
                   const int32_t* __restrict__ cand_rows, const int32_t* __restrict__ cand_cols,
                   int32_t* rows, int32_t* cols) {
  for (int64_t o = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; o < total;
       o += int64_t(gridDim.x) * blockDim.x) {
    const int64_t s = segment_of(sel, n_spaces, o);
    const int32_t e = __ldg(order + __ldg(begin + s) + (o - __ldg(sel + s)));
    const int32_t u = __ldg(cand_rows + e), v = __ldg(cand_cols + e);
    rows[2 * o] = u;
    cols[2 * o] = v;
    rows[2 * o + 1] = v;
    cols[2 * o + 1] = u;
  }
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

int subset_select(int64_t n, int64_t n_chunks, const int64_t* offsets, int64_t n_spaces,
                  const int64_t* space_chunk_host, const int64_t* target_host, uint64_t key,
                  const int32_t* cand_rows, const int32_t* cand_cols, int32_t* rows,
                  int32_t* cols, int max_blocks, cudaStream_t st) {
  for (int64_t s = 0; s < n_spaces; ++s)
    if (space_chunk_host[s] > space_chunk_host[s + 1] || target_host[s] < 0)
      return fail(GSP_ERR_ARG, "subset_select: %s", "bad space table");
  if (space_chunk_host[0] != 0 || space_chunk_host[n_spaces] != n_chunks)
    return fail(GSP_ERR_ARG, "subset_select: %s", "the spaces must cover the chunks");
  std::vector<int64_t> begin(n_spaces + 1), sel(n_spaces + 1, 0);
  Scratch<int64_t> tables(st);
  GSP_CUDA(tables.alloc(3 * (n_spaces + 1)));
  int64_t* d_chunk = tables.get();
  int64_t* d_begin = d_chunk + (n_spaces + 1);
  int64_t* d_sel = d_begin + (n_spaces + 1);
  GSP_CUDA(cudaMemcpyAsync(d_chunk, space_chunk_host, sizeof(int64_t) * (n_spaces + 1),
                           cudaMemcpyHostToDevice, st));
  subset_begin_kernel<<<(unsigned)ceil_div(n_spaces + 1, kThreads), kThreads, 0, st>>>(
      n_spaces, d_chunk, offsets, d_begin);
  GSP_LAUNCH_CHECK("subset_begin");
  GSP_CUDA(cudaMemcpyAsync(begin.data(), d_begin, sizeof(int64_t) * (n_spaces + 1),
                           cudaMemcpyDeviceToHost, st));
  GSP_CUDA(cudaStreamSynchronize(st));
  for (int64_t s = 0; s < n_spaces; ++s) {
    if (begin[s + 1] - begin[s] < target_host[s])
      return fail(GSP_ERR_UNSUPPORTED, "subset_select: %s",
                  "a pair space has fewer candidates than its target; redraw it");
    sel[s + 1] = sel[s] + target_host[s];
  }
  const int64_t n_cand = begin[n_spaces], total = sel[n_spaces];
  if (n_cand >= (int64_t(1) << 31))
    return fail(GSP_ERR_UNSUPPORTED, "subset_select: %s", "2^31 candidates or more");
  if (total == 0) return GSP_OK;
  GSP_CUDA(cudaMemcpyAsync(d_sel, sel.data(), sizeof(int64_t) * (n_spaces + 1),
                           cudaMemcpyHostToDevice, st));
  Scratch<unsigned long long> prio(st);
  Scratch<int32_t> idx(st);
  GSP_CUDA(prio.alloc(2 * n_cand));
  GSP_CUDA(idx.alloc(4 * n_cand));
  unsigned long long* prio_in = prio.get();
  unsigned long long* prio_out = prio_in + n_cand;
  int32_t* pos_a = idx.get();
  int32_t* pos_b = pos_a + n_cand;
  int32_t* spc_in = pos_b + n_cand;
  int32_t* spc_out = spc_in + n_cand;
  const int grid = grid_of(n_cand, max_blocks);
  const int items = (int)n_cand;
  subset_priority_kernel<<<grid, kThreads, 0, st>>>(n_cand, n, cand_rows, cand_cols, key,
                                                    prio_in, pos_a);
  GSP_LAUNCH_CHECK("subset_priority");
  int rc = cub_temp("cub::DeviceRadixSort::SortPairs", st, [&](void* tmp, size_t& bytes) {
    return cub::DeviceRadixSort::SortPairs(tmp, bytes, prio_in, prio_out, pos_a, pos_b, items, 0,
                                           64, st);
  });
  if (rc != GSP_OK) return rc;
  const int32_t* order = pos_b;
  if (n_spaces > 1) {                  // stable: each space keeps the priority order
    int bits = 1;
    while ((int64_t(1) << bits) < n_spaces) ++bits;
    subset_space_kernel<<<grid, kThreads, 0, st>>>(n_cand, n_spaces, d_begin, pos_b, spc_in);
    GSP_LAUNCH_CHECK("subset_space");
    rc = cub_temp("cub::DeviceRadixSort::SortPairs", st, [&](void* tmp, size_t& bytes) {
      return cub::DeviceRadixSort::SortPairs(tmp, bytes, spc_in, spc_out, pos_b, pos_a, items, 0,
                                             bits, st);
    });
    if (rc != GSP_OK) return rc;
    order = pos_a;
  }
  subset_emit_kernel<<<grid_of(total, max_blocks), kThreads, 0, st>>>(
      total, n_spaces, d_sel, d_begin, order, cand_rows, cand_cols, rows, cols);
  GSP_LAUNCH_CHECK("subset_emit");
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
int gsp_subset_select(int64_t n, int64_t n_chunks, const int64_t* offsets, int64_t n_spaces,
                      const int64_t* space_chunk_host, const int64_t* target_host, uint64_t key,
                      const int32_t* cand_rows, const int32_t* cand_cols, int32_t* rows,
                      int32_t* cols, int max_blocks, void* stream) {
  GSP_REQUIRE(n >= 1 && n < (int64_t(1) << 31) && n_chunks >= 0 && offsets, "bad arguments");
  GSP_REQUIRE(n_spaces >= 1 && n_spaces < (int64_t(1) << 31) && space_chunk_host && target_host,
              "bad space table");
  return gsp::subset_select(n, n_chunks, offsets, n_spaces, space_chunk_host, target_host, key,
                            cand_rows, cand_cols, rows, cols, max_blocks, gsp::as_stream(stream));
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
