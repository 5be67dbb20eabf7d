// Kron reduction by random-walk sampling of the Schur complement (kron_reduction(method='walks'),
// pygsp/reduction.py:309-382): the estimator of Durfee, Kyng, Peebles, Rao and Sachdeva,
// "Sampling random spanning trees faster than matrix multiplication" (STOC 2017).
//
// M (n x n, canonical float64 CSR) is an SDDM matrix: off-diagonal entries -w_uv <= 0 and an
// excess e_u = M_uu - sum_v w_uv >= 0 per row, which acts as an edge (u, g) of weight e_u to one
// extra ground vertex g.  K is the kept vertices plus g.  For an edge (u, v) of weight w, walk from
// u until the walk hits K, then from v until it hits K; with endpoints c1, c2 and R the sum of 1/w
// over the steps of both walks, the edge (c1, c2) of weight 1 / (R_u + 1/w + R_v) is a sample
// whose expected Laplacian, summed over the edges, is the Schur complement SC(M, K).  A sample
// (c, g) adds to the diagonal at c; (c, c) and (g, g) add nothing.
//
//   gsp_walk_prep_f64   per row, sequentially in CSR order: prefix[k] = inclusive sum of the
//                       off-diagonal weights -data (the diagonal entry adds 0), total = the row's
//                       sum, and the excess (given, or M_uu - total clamped at 0).  Flags a
//                       negative weight (status bit 1) and an excess below -1e-12 M_uu (bit 2).
//   gsp_schur_walk_f64  one thread per item: (sampled edge e) x samples, then (ground edge of a
//                       removed vertex) x samples.  Item i writes its own slots: 4 triplets for an
//                       edge item, 1 for a ground item (row -1 marks an empty slot), so the output
//                       does not depend on the launch shape.
//
// Draws.  curand_init(key, item, 0); step t of an item (counted across both walks) reads words
// 2 (t mod 2) and 2 (t mod 2) + 1 (lo, hi) of the (t div 2)-th curand4, and
// U = (((hi << 32) | lo) >> 11) 2^-53.  At vertex x the step takes X = U (total_x + e_x): the
// ground when X >= total_x and e_x > 0, else the first CSR position whose prefix exceeds X (a
// zero weight is never taken); the rounding case X >= total_x with e_x = 0 takes the last
// position with a positive weight.  R is one float64 sum in walk order: the steps from u, then
// 1/w (1/e_u for a ground item), then the steps from v.  The sample's value is 1 / (R samples).
//
// Bounds.  An item stops after max_steps steps (status bit 4, nothing emitted); every other loop
// is a CSR row or a binary search over one.  Cost per item: about 2 + steps random reads of the
// CSR arrays; the walks of the eigenvector split are about one step long (DESIGN section 4.23).
#include <curand_kernel.h>

#include "common.cuh"
#include "gspb200.h"

namespace gsp {
namespace {

constexpr int kPrepThreads = 256;
constexpr int kWalkThreads = 128;
constexpr int kGround = -1;   // walk result: the ground vertex
constexpr int kCapped = -2;   // walk result: max_steps reached

__global__ void __launch_bounds__(kPrepThreads)
walk_prep_kernel(int64_t n, const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                 const double* __restrict__ data, const double* __restrict__ excess_in,
                 double* __restrict__ prefix, double* __restrict__ total,
                 double* __restrict__ excess, int32_t* __restrict__ status) {
  const int64_t u = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (u >= n) return;
  double acc = 0.0, diag = 0.0;
  int flags = 0;
  const int64_t e = indptr[u + 1];
  for (int64_t k = indptr[u]; k < e; ++k) {
    const double m = data[k];
    if (indices[k] == u) {
      diag = m;
    } else {
      if (m > 0.0) flags |= 1;
      acc += -m;
    }
    prefix[k] = acc;
  }
  total[u] = acc;
  double ex;
  if (excess_in) {
    ex = excess_in[u];
  } else {
    ex = diag - acc;
    if (ex < -1e-12 * diag) flags |= 2;
  }
  excess[u] = ex > 0.0 ? ex : 0.0;
  if (flags) atomicOr(status, flags);
}

// first position p in [b, e) with prefix[p] > x (strict) or >= x, e if none
template <bool STRICT>
__device__ __forceinline__ int64_t search(const double* __restrict__ prefix, int64_t b, int64_t e,
                                          double x) {
  while (b < e) {
    const int64_t mid = b + ((e - b) >> 1);
    const double p = __ldg(prefix + mid);
    if (STRICT ? p > x : p >= x) e = mid; else b = mid + 1;
  }
  return b;
}

struct Walker {
  const int32_t* indptr;
  const int32_t* indices;
  const double* data;
  const double* prefix;
  const double* total;
  const double* excess;
  const int32_t* slot;
  int64_t max_steps;
  curandStatePhilox4_32_10_t state;
  uint4 draw;
  int64_t t;

  // walk from x until a kept vertex (its kept index) or the ground (kGround); kCapped at
  // max_steps.  Adds 1/w of every step to R, in order.
  __device__ int walk(int x, double& R) {
    for (;;) {
      const int s = __ldg(slot + x);
      if (s < 0) return -1 - s;
      if (t >= max_steps) return kCapped;
      if ((t & 1) == 0) draw = curand4(&state);
      const uint32_t lo = (t & 1) ? draw.z : draw.x;
      const uint32_t hi = (t & 1) ? draw.w : draw.y;
      ++t;
      const double U = double(((uint64_t(hi) << 32) | lo) >> 11) * 0x1p-53;
      const double tot = __ldg(total + x), ex = __ldg(excess + x);
      const double X = U * (tot + ex);
      if (X >= tot && ex > 0.0) {
        R += 1.0 / ex;
        return kGround;
      }
      const int64_t b = __ldg(indptr + x), e = __ldg(indptr + x + 1);
      int64_t p = search<true>(prefix, b, e, X);
      if (p == e) p = search<false>(prefix, b, e, tot);   // rounding: the last positive weight
      if (p == e) return kCapped;                          // no positive weight: cannot happen
      R += 1.0 / -__ldg(data + p);
      x = __ldg(indices + p);
    }
  }
};

__global__ void __launch_bounds__(kWalkThreads)
schur_walk_kernel(Walker base, int64_t n_edges, const int32_t* __restrict__ eu,
                  const int32_t* __restrict__ ev, const double* __restrict__ ew, int64_t n_ground,
                  const int32_t* __restrict__ gu, int samples, uint64_t key,
                  int32_t* __restrict__ rows, int32_t* __restrict__ cols, double* __restrict__ vals,
                  int32_t* __restrict__ steps, int32_t* __restrict__ status) {
  const int64_t edge_items = n_edges * samples;
  const int64_t item = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (item >= edge_items + n_ground * samples) return;
  Walker w = base;
  w.t = 0;
  curand_init(key, uint64_t(item), 0ull, &w.state);
  const bool is_edge = item < edge_items;
  int a, b;
  double inv_w;
  int64_t out;
  int nslots;
  if (is_edge) {
    const int64_t e = item / samples;
    a = eu[e];
    b = ev[e];
    inv_w = 1.0 / ew[e];
    out = 4 * item;
    nslots = 4;
  } else {
    const int64_t g = (item - edge_items) / samples;
    a = gu[g];
    b = -1;
    inv_w = 1.0 / __ldg(w.excess + a);
    out = 4 * edge_items + (item - edge_items);
    nslots = 1;
  }
  double R = 0.0;
  int c1 = w.walk(a, R), c2 = kGround;
  if (c1 != kCapped) {
    R += inv_w;
    if (is_edge) c2 = w.walk(b, R);
  }
  if (steps) steps[item] = int32_t(w.t < INT32_MAX ? w.t : INT32_MAX);
  int32_t r[4] = {-1, -1, -1, -1}, c[4] = {-1, -1, -1, -1};
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  if (c1 == kCapped || c2 == kCapped) {
    atomicOr(status, 4);
  } else if (c1 != c2) {
    const double val = 1.0 / (R * double(samples));
    if (c1 == kGround || c2 == kGround) {
      const int k = c1 == kGround ? c2 : c1;
      r[0] = c[0] = k;
      v[0] = val;
    } else {
      r[0] = c1; c[0] = c2; v[0] = -val;
      r[1] = c2; c[1] = c1; v[1] = -val;
      r[2] = c1; c[2] = c1; v[2] = val;
      r[3] = c2; c[3] = c2; v[3] = val;
    }
  }
  for (int q = 0; q < nslots; ++q) {
    rows[out + q] = r[q];
    cols[out + q] = c[q];
    vals[out + q] = v[q];
  }
}

}  // namespace

int walk_prep(int64_t n, const int32_t* indptr, const int32_t* indices, const double* data,
              const double* excess_in, double* prefix, double* total, double* excess,
              int32_t* status, cudaStream_t st) {
  if (n == 0) return GSP_OK;
  walk_prep_kernel<<<(unsigned)ceil_div(n, kPrepThreads), kPrepThreads, 0, st>>>(
      n, indptr, indices, data, excess_in, prefix, total, excess, status);
  GSP_LAUNCH_CHECK("walk_prep");
  return GSP_OK;
}

int schur_walk(const Walker& base, int64_t n_edges, const int32_t* eu, const int32_t* ev,
               const double* ew, int64_t n_ground, const int32_t* gu, int samples, uint64_t key,
               int32_t* rows, int32_t* cols, double* vals, int32_t* steps, int32_t* status,
               cudaStream_t st) {
  const int64_t items = (n_edges + n_ground) * samples;
  if (items == 0) return GSP_OK;
  schur_walk_kernel<<<(unsigned)ceil_div(items, kWalkThreads), kWalkThreads, 0, st>>>(
      base, n_edges, eu, ev, ew, n_ground, gu, samples, key, rows, cols, vals, steps, status);
  GSP_LAUNCH_CHECK("schur_walk");
  return GSP_OK;
}

}  // namespace gsp

extern "C" {
int gsp_walk_prep_f64(int64_t n, const int32_t* indptr, const int32_t* indices, const double* data,
                      const double* excess_in, double* prefix, double* total, double* excess,
                      int32_t* status, void* stream) {
  GSP_REQUIRE(n >= 0 && n < (int64_t(1) << 31), "bad arguments");
  GSP_REQUIRE(n == 0 || (indptr && indices && data && prefix && total && excess && status),
              "no buffer");
  return gsp::walk_prep(n, indptr, indices, data, excess_in, prefix, total, excess, status,
                        gsp::as_stream(stream));
}
int gsp_schur_walk_f64(const int32_t* indptr, const int32_t* indices, const double* data,
                       const double* prefix, const double* total, const double* excess,
                       const int32_t* slot, int64_t n_edges, const int32_t* eu, const int32_t* ev,
                       const double* ew, int64_t n_ground, const int32_t* gu, int64_t samples,
                       uint64_t key, int64_t max_steps, int32_t* rows, int32_t* cols,
                       double* vals, int32_t* steps, int32_t* status, void* stream) {
  GSP_REQUIRE(n_edges >= 0 && n_ground >= 0 && samples >= 1 && samples < (int64_t(1) << 31) &&
                  max_steps >= 0,
              "bad arguments");
  GSP_REQUIRE((n_edges + n_ground) < (int64_t(1) << 31) / samples &&
                  4 * n_edges * samples + n_ground * samples < (int64_t(1) << 31),
              "too many items");
  GSP_REQUIRE(n_edges + n_ground == 0 ||
                  (indptr && indices && data && prefix && total && excess && slot && rows &&
                   cols && vals && status),
              "no buffer");
  GSP_REQUIRE(n_edges == 0 || (eu && ev && ew), "no edge buffer");
  GSP_REQUIRE(n_ground == 0 || gu, "no ground buffer");
  gsp::Walker base{indptr, indices, data, prefix, total, excess, slot, max_steps, {}, {}, 0};
  return gsp::schur_walk(base, n_edges, eu, ev, ew, n_ground, gu, (int)samples, key, rows, cols,
                         vals, steps, status, gsp::as_stream(stream));
}
}
