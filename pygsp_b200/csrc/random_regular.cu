// Random regular graphs (pygsp/graphs/randomregular.py): stub pairing on the device.
//
// Replaces the sequential lil_matrix loop of randomregular.py:62-98 -> gsp_random_regular, and
// writes the complement of a sampled graph straight into CSR -> gsp_random_regular_complement.
//
// A k-regular graph on n vertices pairs n k stubs (stub p belongs to vertex p mod n, the order of
// the reference's kron(ones(k), arange(n))).  Every draw comes from a Philox4x32-10 stream of the
// caller's key whose subsequence is (attempt << 32) | phase: phase r < 2^32 - 2 is bulk round r,
// GSPB200_RR_TAIL_STREAM the tail, GSPB200_RR_SWITCH_STREAM the switches; the offset is a pool
// position or a draw number.  No draw depends on a thread or block id, so the graph is a function of
// (key, n, k, max_iter) alone and a serial restatement reproduces it bit for bit.
//
// Attempt a:
//   * Bulk rounds, while the pool holds more than GSPB200_RR_TAIL_STUBS stubs.  Stub p of the pool
//     gets the 64-bit priority (x << 32) | y of curand4 block p of round r; one stable radix sort
//     orders the pool, positions (2i, 2i + 1) form pair i.  Pair i is legal when u != v and {u, v}
//     is not in the edge table as it stood at the start of the round (a check launch that only
//     reads it); a claim launch then inserts the legal pairs' keys and keeps the lowest pair index
//     per key (atomicMin), and exactly that pair is accepted.  Accepted edges go to the edge list
//     at scanned offsets, rejected stubs are compacted stably into the next pool.
//   * The tail: one CTA.  Thread 0 runs the reference's rule on the pool held in shared memory:
//     two uniform positions i1 = mulhi(u1, P), i2 = mulhi(u2, P) per curand4 draw, the pair
//     accepted when legal, both stubs swap-removed (larger position first).  After
//     GSPB200_RR_CHECK_AFTER rejections in a row the whole CTA checks every pair of the pool
//     exactly; no legal pair means the pool is stuck.  At most GSPB200_RR_TAIL_DRAWS draws.
//   * A stuck pool or the draw cap ends the attempt; the next one starts from scratch.  The last
//     attempt instead places each remaining stub pair (a, b), in pool order, by a switch: draw an
//     edge e = mulhi(u, E) of the list and an orientation (x, y), until x, y not in {a, b},
//     {a, x} and {b, y} are not edges; then edge e becomes (a, x) and (b, y) is appended.  A pair
//     whose GSPB200_RR_SWITCH_DRAWS draws all fail stops the switches: the graph stays partial.
//
// The edge table is open addressing with linear probing over canonical keys (min << 32) | max,
// capacity a power of two >= stubs + 2 GSPB200_RR_TAIL_STUBS, so its load stays below one half
// (switches leave tombstones).  Every probe loop is bounded by the capacity.
#include <cub/cub.cuh>
#include <curand_kernel.h>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {
namespace {

constexpr int kThreads = 256;
constexpr int kTailStubs = GSPB200_RR_TAIL_STUBS;
constexpr int kCheckAfter = GSPB200_RR_CHECK_AFTER;
constexpr long long kTailDraws = GSPB200_RR_TAIL_DRAWS;
constexpr int kSwitchDraws = GSPB200_RR_SWITCH_DRAWS;
constexpr int kMaxRounds = GSPB200_RR_MAX_ROUNDS;
constexpr int kCheckChunk = 8;                      // pairs per thread between two votes
constexpr uint64_t kEmpty = ~0ull, kTomb = ~0ull - 1;

// tail status: 0 complete, 1 failed attempt, 2 partial graph kept
constexpr int kDone = 0, kFailed = 1, kPartial = 2;

__device__ __forceinline__ uint64_t edge_key(int32_t u, int32_t v) {
  const uint32_t a = (uint32_t)min(u, v), b = (uint32_t)max(u, v);
  return (uint64_t(a) << 32) | b;
}

__device__ __forceinline__ uint64_t slot_of(uint64_t e, uint64_t mask) {
  e ^= e >> 33;
  e *= 0xff51afd7ed558ccdull;
  e ^= e >> 33;
  e *= 0xc4ceb9fe1a85ec53ull;
  e ^= e >> 33;
  return e & mask;
}

__device__ bool table_has(const unsigned long long* keys, uint64_t mask, uint64_t e) {
  uint64_t s = slot_of(e, mask);
  for (uint64_t i = 0; i <= mask; ++i, s = (s + 1) & mask) {
    const uint64_t k = keys[s];
    if (k == e) return true;
    if (k == kEmpty) return false;
  }
  return false;
}

// single-threaded insert of a key known to be absent (tail and switches)
__device__ void table_put(unsigned long long* keys, uint64_t mask, uint64_t e) {
  uint64_t s = slot_of(e, mask);
  for (uint64_t i = 0; i <= mask; ++i, s = (s + 1) & mask) {
    if (keys[s] == kEmpty || keys[s] == kTomb) {
      keys[s] = e;
      return;
    }
  }
}

__device__ void table_erase(unsigned long long* keys, uint64_t mask, uint64_t e) {
  uint64_t s = slot_of(e, mask);
  for (uint64_t i = 0; i <= mask; ++i, s = (s + 1) & mask) {
    if (keys[s] == e) {
      keys[s] = kTomb;
      return;
    }
    if (keys[s] == kEmpty) return;
  }
}

__device__ __forceinline__ uint4 draw4(uint64_t key, uint64_t sub, uint64_t t) {
  curandStatePhilox4_32_10_t state;
  curand_init(key, sub, 4ull * t, &state);
  return curand4(&state);
}

__device__ __forceinline__ uint32_t mulhi_n(uint32_t hi, uint32_t lo, uint32_t n) {
  return (uint32_t)__umul64hi((uint64_t(hi) << 32) | lo, n);
}

__global__ void __launch_bounds__(kThreads)
rr_init_pool_kernel(int64_t stubs, int64_t n, int32_t* pool) {
  for (int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; p < stubs;
       p += int64_t(gridDim.x) * blockDim.x)
    pool[p] = (int32_t)(p % n);
}

__global__ void __launch_bounds__(kThreads)
rr_priority_kernel(int64_t P, uint64_t key, uint64_t sub, unsigned long long* prio) {
  for (int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; p < P;
       p += int64_t(gridDim.x) * blockDim.x) {
    const uint4 r = draw4(key, sub, (uint64_t)p);
    prio[p] = (uint64_t(r.x) << 32) | r.y;
  }
}

// state[i] = 1 when pair i is legal against the table as it stands (nothing is written to it)
__global__ void __launch_bounds__(kThreads)
rr_check_kernel(int64_t pairs, const int32_t* __restrict__ pool,
                const unsigned long long* __restrict__ keys, uint64_t mask, int32_t* state) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < pairs;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int32_t u = __ldg(pool + 2 * i), v = __ldg(pool + 2 * i + 1);
    state[i] = u != v && !table_has(keys, mask, edge_key(u, v));
  }
}

// legal pairs insert their key; the lowest pair index per key becomes its owner
__global__ void __launch_bounds__(kThreads)
rr_claim_kernel(int64_t pairs, const int32_t* __restrict__ pool, const int32_t* __restrict__ state,
                unsigned long long* keys, int32_t* owner, uint64_t mask, int64_t* slot) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < pairs;
       i += int64_t(gridDim.x) * blockDim.x) {
    if (!__ldg(state + i)) continue;
    const uint64_t e = edge_key(__ldg(pool + 2 * i), __ldg(pool + 2 * i + 1));
    uint64_t s = slot_of(e, mask);
    for (uint64_t t = 0; t <= mask; ++t, s = (s + 1) & mask) {
      const unsigned long long k = atomicCAS(keys + s, kEmpty, e);
      if (k == kEmpty || k == e) {
        atomicMin(owner + s, (int32_t)i);
        slot[i] = (int64_t)s;
        break;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
rr_resolve_kernel(int64_t pairs, const int32_t* __restrict__ owner,
                  const int64_t* __restrict__ slot, int32_t* state) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < pairs;
       i += int64_t(gridDim.x) * blockDim.x)
    if (state[i]) state[i] = __ldg(owner + __ldg(slot + i)) == (int32_t)i;
}

// off: inclusive scan of the accepted flags (off[-1] = 0 implied for i = 0)
__global__ void __launch_bounds__(kThreads)
rr_emit_kernel(int64_t pairs, const int32_t* __restrict__ pool, const int32_t* __restrict__ off,
               int64_t E, int32_t* eu, int32_t* ev, int32_t* next) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < pairs;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int32_t u = __ldg(pool + 2 * i), v = __ldg(pool + 2 * i + 1);
    const int32_t before = i ? __ldg(off + i - 1) : 0;
    if (__ldg(off + i) != before) {
      eu[E + before] = u;
      ev[E + before] = v;
    } else {
      const int64_t r = i - before;
      next[2 * r] = u;
      next[2 * r + 1] = v;
    }
  }
}

// The tail of one attempt (see the file comment); one CTA of kThreads.  io[0] = E on entry and
// exit; io[1] = status.
__global__ void __launch_bounds__(kThreads)
rr_tail_kernel(int P0, const int32_t* __restrict__ pool_in, uint64_t key, uint64_t attempt,
               int last, unsigned long long* keys, uint64_t mask, int32_t* eu, int32_t* ev,
               int64_t* io) {
  __shared__ int32_t pool[kTailStubs];
  __shared__ int s_cmd, s_P;
  enum { kRun = 0, kCheck = 1, kEnd = 2 };
  for (int p = threadIdx.x; p < P0; p += blockDim.x) pool[p] = pool_in[p];
  const uint64_t sub = attempt << 32;
  int64_t E = io[0];
  long long t = 0;
  int P = P0;
  __syncthreads();
  while (true) {
    if (threadIdx.x == 0) {
      int rej = 0;
      while (P > 0 && rej < kCheckAfter && t < kTailDraws) {
        const uint4 r = draw4(key, sub | GSPB200_RR_TAIL_STREAM, (uint64_t)t++);
        const int i1 = (int)mulhi_n(r.x, r.y, (uint32_t)P);
        const int i2 = (int)mulhi_n(r.z, r.w, (uint32_t)P);
        const int32_t v1 = pool[i1], v2 = pool[i2];
        if (v1 != v2 && !table_has(keys, mask, edge_key(v1, v2))) {
          table_put(keys, mask, edge_key(v1, v2));
          eu[E] = v1;
          ev[E] = v2;
          ++E;
          pool[max(i1, i2)] = pool[P - 1];
          --P;
          pool[min(i1, i2)] = pool[P - 1];
          --P;
          rej = 0;
        } else {
          ++rej;
        }
      }
      s_cmd = (P == 0 || t >= kTailDraws) ? kEnd : kCheck;
      s_P = P;
    }
    __syncthreads();
    if (s_cmd == kEnd) break;
    // exact check: is any pair of positions i < j of the pool legal?
    const int n = s_P;
    const int64_t cells = int64_t(n) * n;
    bool found = false;
    for (int64_t base = 0; base < cells && !found; base += int64_t(kThreads) * kCheckChunk) {
      bool mine = false;
      for (int c = 0; c < kCheckChunk; ++c) {
        const int64_t q = base + int64_t(c) * kThreads + threadIdx.x;
        if (q >= cells) break;
        const int i = (int)(q / n), j = (int)(q % n);
        if (i < j && pool[i] != pool[j] && !table_has(keys, mask, edge_key(pool[i], pool[j])))
          mine = true;
      }
      found = __syncthreads_or(mine);
    }
    if (!found) break;                                // stuck
  }
  if (threadIdx.x != 0) return;
  int status = P == 0 ? kDone : kFailed;
  if (P > 0 && last) {
    status = kDone;
    long long ts = 0;
    for (int p = 0; p < P && status == kDone; p += 2) {
      const int32_t a = pool[p], b = pool[p + 1];
      status = kPartial;
      for (int d = 0; d < kSwitchDraws && E > 0; ++d) {
        const uint4 r = draw4(key, sub | GSPB200_RR_SWITCH_STREAM, (uint64_t)ts++);
        const int64_t e = (int64_t)__umul64hi((uint64_t(r.x) << 32) | r.y, (uint64_t)E);
        const bool flip = r.z & 1;
        const int32_t x = flip ? ev[e] : eu[e], y = flip ? eu[e] : ev[e];
        if (x == a || x == b || y == a || y == b) continue;
        if (table_has(keys, mask, edge_key(a, x)) || table_has(keys, mask, edge_key(b, y)))
          continue;
        table_erase(keys, mask, edge_key(x, y));
        table_put(keys, mask, edge_key(a, x));
        table_put(keys, mask, edge_key(b, y));
        eu[e] = a;
        ev[e] = x;
        eu[E] = b;
        ev[E] = y;
        ++E;
        status = kDone;
        break;
      }
    }
  }
  io[0] = E;
  io[1] = status;
}

__global__ void __launch_bounds__(kThreads)
rr_coo_kernel(int64_t E, const int32_t* __restrict__ eu, const int32_t* __restrict__ ev,
              int32_t* rows, int32_t* cols) {
  for (int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; e < E;
       e += int64_t(gridDim.x) * blockDim.x) {
    const int32_t u = __ldg(eu + e), v = __ldg(ev + e);
    rows[2 * e] = u;
    cols[2 * e] = v;
    rows[2 * e + 1] = v;
    cols[2 * e + 1] = u;
  }
}

__global__ void __launch_bounds__(kThreads)
rr_complement_indptr_kernel(int64_t n, const int32_t* __restrict__ indptr, int32_t* out) {
  for (int64_t u = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; u <= n;
       u += int64_t(gridDim.x) * blockDim.x)
    out[u] = (int32_t)(u * (n - 1) - __ldg(indptr + u));
}

// Entry j of complement row u is the j-th vertex outside X = {u} U N(u) (sorted, m = |X|):
// v = j + #{i : X[i] - i <= j}, X[i] - i being non-decreasing.
__global__ void __launch_bounds__(kThreads)
rr_complement_fill_kernel(int64_t n, int64_t nnz, const int32_t* __restrict__ indptr,
                          const int32_t* __restrict__ indices, const int32_t* __restrict__ out_ptr,
                          int32_t* out) {
  for (int64_t q = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; q < nnz;
       q += int64_t(gridDim.x) * blockDim.x) {
    int64_t lo = 0, hi = n - 1;                       // row: last u with out_ptr[u] <= q
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) >> 1;
      if (__ldg(out_ptr + mid) <= q) lo = mid; else hi = mid - 1;
    }
    const int32_t u = (int32_t)lo;
    const int32_t j = (int32_t)(q - __ldg(out_ptr + u));
    const int32_t* nb = indices + __ldg(indptr + u);
    const int32_t deg = __ldg(indptr + u + 1) - __ldg(indptr + u);
    int32_t pu = 0, ph = deg;                         // position of u among its neighbours
    while (pu < ph) {
      const int32_t mid = (pu + ph) >> 1;
      if (__ldg(nb + mid) < u) pu = mid + 1; else ph = mid;
    }
    int32_t a = 0, b = deg + 1;                       // count of i in [0, deg] with X[i] - i <= j
    while (a < b) {
      const int32_t i = (a + b) >> 1;
      const int32_t x = i < pu ? __ldg(nb + i) : (i == pu ? u : __ldg(nb + i - 1));
      if (x - i <= j) a = i + 1; else b = i;
    }
    out[q] = j + a;
  }
}

int grid_of(int64_t work, int max_blocks) {
  int64_t g = ceil_div(work, kThreads);
  if (max_blocks > 0 && g > max_blocks) g = max_blocks;
  const int64_t cap = int64_t(sm_count()) * 32;
  return (int)std::max<int64_t>(1, std::min(g, cap));
}

}  // namespace

int random_regular(int64_t n, int64_t k, int max_iter, uint64_t key, int32_t* rows, int32_t* cols,
                   int max_blocks, int* attempts, int* rounds, int64_t* entries, cudaStream_t st) {
  *attempts = 0;
  *rounds = 0;
  *entries = 0;
  const int64_t stubs = n * k;
  if (stubs == 0) return GSP_OK;
  uint64_t cap = 1024;
  while (cap < uint64_t(stubs) + 2 * kTailStubs) cap <<= 1;
  const uint64_t mask = cap - 1;
  const int64_t pairs_max = stubs / 2;
  Scratch<unsigned long long> table(st), prio(st);
  Scratch<int32_t> owner(st), pools(st), pair_i32(st), edges(st);
  Scratch<int64_t> slot(st), io(st);
  GSP_CUDA(table.alloc(cap));
  GSP_CUDA(owner.alloc(cap));
  GSP_CUDA(pools.alloc(2 * stubs));
  GSP_CUDA(edges.alloc(2 * pairs_max));
  GSP_CUDA(io.alloc(2));
  const bool bulk = stubs > kTailStubs;
  if (bulk) {
    GSP_CUDA(prio.alloc(2 * stubs));
    GSP_CUDA(pair_i32.alloc(2 * pairs_max));
    GSP_CUDA(slot.alloc(pairs_max));
  }
  int32_t* eu = edges.get();
  int32_t* ev = eu + pairs_max;
  int64_t E = 0;
  int total_rounds = 0;
  int64_t host_io[2] = {0, kFailed};
  for (int a = 0; a < max_iter; ++a) {
    GSP_CUDA(cudaMemsetAsync(table.get(), 0xff, sizeof(uint64_t) * cap, st));
    // owners start at 0x7f7f7f7f, above every pair index (pairs < 2^30)
    GSP_CUDA(cudaMemsetAsync(owner.get(), 0x7f, sizeof(int32_t) * cap, st));
    int32_t* pool = pools.get();
    int32_t* spare = pool + stubs;
    rr_init_pool_kernel<<<grid_of(stubs, max_blocks), kThreads, 0, st>>>(stubs, n, pool);
    GSP_LAUNCH_CHECK("rr_init_pool");
    int64_t P = stubs;
    E = 0;
    for (int r = 0; P > kTailStubs; ++r) {
      if (r == kMaxRounds)
        return fail(GSP_ERR_UNSUPPORTED, "random_regular: the pool is still above %s stubs after "
                    "%s rounds", "GSPB200_RR_TAIL_STUBS", "GSPB200_RR_MAX_ROUNDS");
      const int64_t pairs = P / 2;
      const int grid = grid_of(P, max_blocks);
      unsigned long long* pr_in = prio.get();
      unsigned long long* pr_out = pr_in + stubs;
      rr_priority_kernel<<<grid, kThreads, 0, st>>>(P, key, (uint64_t(a) << 32) | uint64_t(r),
                                                    pr_in);
      GSP_LAUNCH_CHECK("rr_priority");
      int rc = cub_temp("cub::DeviceRadixSort::SortPairs", st, [&](void* tmp, size_t& bytes) {
        return cub::DeviceRadixSort::SortPairs(tmp, bytes, pr_in, pr_out, pool, spare, (int)P, 0, 64,
                                               st);
      });
      if (rc != GSP_OK) return rc;
      std::swap(pool, spare);                          // pool: the sorted stubs
      int32_t* state = pair_i32.get();
      int32_t* off = state + pairs_max;
      const int pgrid = grid_of(pairs, max_blocks);
      rr_check_kernel<<<pgrid, kThreads, 0, st>>>(pairs, pool, table.get(), mask, state);
      GSP_LAUNCH_CHECK("rr_check");
      rr_claim_kernel<<<pgrid, kThreads, 0, st>>>(pairs, pool, state, table.get(), owner.get(),
                                                  mask, slot.get());
      GSP_LAUNCH_CHECK("rr_claim");
      rr_resolve_kernel<<<pgrid, kThreads, 0, st>>>(pairs, owner.get(), slot.get(), state);
      GSP_LAUNCH_CHECK("rr_resolve");
      rc = cub_temp("cub::DeviceScan::InclusiveSum", st, [&](void* tmp, size_t& bytes) {
        return cub::DeviceScan::InclusiveSum(tmp, bytes, state, off, (int)pairs, st);
      });
      if (rc != GSP_OK) return rc;
      rr_emit_kernel<<<pgrid, kThreads, 0, st>>>(pairs, pool, off, E, eu, ev, spare);
      GSP_LAUNCH_CHECK("rr_emit");
      std::swap(pool, spare);                          // pool: the rejected stubs
      int32_t accepted = 0;
      GSP_CUDA(cudaMemcpyAsync(&accepted, off + pairs - 1, sizeof(int32_t),
                               cudaMemcpyDeviceToHost, st));
      GSP_CUDA(cudaStreamSynchronize(st));
      E += accepted;
      P -= 2 * int64_t(accepted);
      ++total_rounds;
    }
    host_io[0] = E;
    GSP_CUDA(cudaMemcpyAsync(io.get(), host_io, sizeof(int64_t), cudaMemcpyHostToDevice, st));
    rr_tail_kernel<<<1, kThreads, 0, st>>>((int)P, pool, key, (uint64_t)a, a == max_iter - 1,
                                           table.get(), mask, eu, ev, io.get());
    GSP_LAUNCH_CHECK("rr_tail");
    GSP_CUDA(cudaMemcpyAsync(host_io, io.get(), 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    GSP_CUDA(cudaStreamSynchronize(st));
    E = host_io[0];
    *attempts = a + 1;
    if (host_io[1] != kFailed) break;
  }
  *rounds = total_rounds;
  if (E > 0) {
    rr_coo_kernel<<<grid_of(E, max_blocks), kThreads, 0, st>>>(E, eu, ev, rows, cols);
    GSP_LAUNCH_CHECK("rr_coo");
  }
  *entries = 2 * E;
  return GSP_OK;
}

int random_regular_complement(int64_t n, int64_t out_nnz, const int32_t* indptr,
                              const int32_t* indices, int32_t* out_indptr, int32_t* out_indices,
                              cudaStream_t st) {
  rr_complement_indptr_kernel<<<grid_of(n + 1, 0), kThreads, 0, st>>>(n, indptr, out_indptr);
  GSP_LAUNCH_CHECK("rr_complement_indptr");
  if (out_nnz == 0) return GSP_OK;
  rr_complement_fill_kernel<<<grid_of(out_nnz, 0), kThreads, 0, st>>>(n, out_nnz, indptr, indices,
                                                                      out_indptr, out_indices);
  GSP_LAUNCH_CHECK("rr_complement_fill");
  return GSP_OK;
}

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {
int gsp_random_regular(int64_t n, int64_t k, int max_iter, uint64_t key, int32_t* rows,
                       int32_t* cols, int max_blocks, int* attempts_host_out,
                       int* rounds_host_out, int64_t* entries_host_out, void* stream) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31) && k >= 0 && (k < n || k == 0) && max_iter >= 1 &&
                  attempts_host_out && rounds_host_out && entries_host_out,
              "bad arguments");
  GSP_REQUIRE(n * k < (int64_t(1) << 31) && (n * k) % 2 == 0, "n k must be even and below 2^31");
  GSP_REQUIRE(n * k == 0 || (rows && cols), "no output");
  return gsp::random_regular(n, k, max_iter, key, rows, cols, max_blocks, attempts_host_out,
                             rounds_host_out, entries_host_out, gsp::as_stream(stream));
}
int gsp_random_regular_complement(int64_t n, int64_t nnz, const int32_t* indptr,
                                  const int32_t* indices, int32_t* out_indptr,
                                  int32_t* out_indices, void* stream) {
  GSP_REQUIRE(n >= 1 && n < (int64_t(1) << 31) && nnz >= 0 && nnz < (int64_t(1) << 31) &&
                  nnz <= n * (n - 1) && indptr && out_indptr && (nnz == 0 || out_indices),
              "bad arguments");
  return gsp::random_regular_complement(n, nnz, indptr, indices, out_indptr, out_indices,
                                        gsp::as_stream(stream));
}
}
