// Proximal operator of graph total variation by FISTA on the dual (fast gradient projection).
//
// Replaces pygsp/optimization.py:24-103 (prox_tv), which hands
//   min_z  1/2 ||x - z||^2 + gamma ||D^T A z||_1
// to pyunlocbox's norm_l1 prox and cannot run as written.  With K = D^T A, K* = A* D, the dual
// variable u in [-1, 1]^(Ne x Nsig), the bound nu_bar >= ||K||^2 and tau = 1 / (gamma nu_bar),
// iteration k is two launches:
//
//   vertex  z_k = x - gamma D u_k       (cheby_step, non-first form: alpha = -gamma, beta = 0,
//                                        gamma = 1, x_old = x; the A = None path)
//   edge    g_k = D^T w  (w = z_k, or A z_k), in double from the two entries of each D^T row;
//           partial sums of |g_k|, |g_k| - u_k g_k and, over a grid-stride slice of the vertices,
//           (x - z_k)^2;
//           v = u_k + b (u_k - u_{k-1}),  K v = (1 + b) g_k - b g_{k-1}  (linearity: one product)
//           u_{k+1} = clip(v + tau K v, -1, 1) over u_{k-1}, g_k over g_{k-1};
//           the last block to finish reduces the partials in block order, records
//           P_k = 1/2 ||x - z_k||^2 + gamma ||g_k||_1 and gap_k = gamma sum(|g_k| - u_k g_k), and
//           applies the stop rule.
//
// Once the rule has fired every later edge launch returns at once, so u_k of the stopping
// iteration stays in U2 block k % 2.  Vertex launches enqueued after the stop still overwrite z;
// the caller recomputes z_k from u_k with one more vertex pass (gsp_prox_tv_primal_*), which
// runs the same kernel on the same operands and so gives the same bits.
//
// Every element's arithmetic is the same whatever Nsig and the lane packing, so column j of a
// block follows the single-column iteration bit for bit; only the sums (and so the stop test)
// see the other columns.  The scratch has the FISTA layout of csrc/reduce.cuh; its history holds
// P_k and gap_k at 2 k and 2 k + 1.
#include <math.h>

#include "reduce.cuh"
#include "step.cuh"

namespace gsp {

enum { kTvRunning = 0, kTvRtol = 1, kTvMaxit = 2 };

// One edge pass (k = it): see the file comment.  V == 1 runs a sub-warp of w = 2^ceil(log2 Nsig)
// lanes per edge (32 / w edges per warp); V > 1 a warp per edge, V columns per lane in flight,
// in chunks of 32 V columns.  Uo holds u_{k-1} on entry and u_{k+1} on exit, Gk g_{k-1} and g_k:
// each element is read before the same thread overwrites it.
template <typename T, int V>
__global__ void __launch_bounds__(kThreads)
tv_edge_kernel(int64_t n, int64_t ne, int nsig, int w, const int32_t* __restrict__ dt_indptr,
               const int32_t* __restrict__ dt_indices, const T* __restrict__ dt_data,
               const T* __restrict__ wv, const T* __restrict__ x, const T* __restrict__ z,
               const T* __restrict__ Uk, T* Uo, T* Gk, double gamma, double tau, double tol,
               int it, int maxit, double* scal) {
  if (scal[1] != 0.0) return;                      // stopped at an earlier iteration
  const double t = it == 0 ? 1.0 : scal[0];
  const double tn = (1.0 + sqrt(1.0 + 4.0 * t * t)) / 2.0;
  const double b = (t - 1.0) / tn;
  const int lane = threadIdx.x % w, grp = threadIdx.x / w, epb = kThreads / w;
  double a_l1 = 0, a_gap = 0, a_v = 0;
  for (int64_t e0 = int64_t(blockIdx.x) * epb; e0 < ne; e0 += int64_t(gridDim.x) * epb) {
    const int64_t e = e0 + grp;
    if (e >= ne) continue;
    // a row of D^T holds two entries, or none for a self-loop (csrc/difference.cu)
    const int p = __ldg(dt_indptr + e);
    const bool pair = __ldg(dt_indptr + e + 1) > p;
    int64_t s0 = 0, s1 = 0;
    double v0 = 0, v1 = 0;
    if (pair) {
      s0 = int64_t(__ldg(dt_indices + p)) * nsig;
      s1 = int64_t(__ldg(dt_indices + p + 1)) * nsig;
      v0 = double(__ldg(dt_data + p));
      v1 = double(__ldg(dt_data + p + 1));
    }
    for (int cb = 0; cb < nsig; cb += w * V) {
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const int c = cb + lane + v * w;
        if (c >= nsig) continue;
        const int64_t i = e * nsig + c;
        // explicit roundings: no fma, so that the two products of a constant signal cancel
        const double g = pair ? __dmul_rn(v0, double(__ldg(wv + s0 + c))) +
                                    __dmul_rn(v1, double(__ldg(wv + s1 + c)))
                              : 0.0;
        const double uk = double(__ldg(Uk + i)), up = double(Uo[i]), gp = double(Gk[i]);
        a_l1 += fabs(g);
        a_gap += fabs(g) - uk * g;
        const double ve = uk + b * (uk - up);
        const double kv = (1.0 + b) * g - b * gp;
        Gk[i] = T(g);
        Uo[i] = T(fmin(1.0, fmax(-1.0, ve + tau * kv)));
      }
    }
  }
  const int64_t nv = n * nsig;
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < nv;
       i += int64_t(gridDim.x) * kThreads) {
    const double d = double(__ldg(x + i)) - double(__ldg(z + i));
    a_v += d * d;
  }

  const double sums[3] = {a_l1, a_gap, a_v};
  fista_last_block(sums, scal, [&](const double (&tot)[3]) {   // objective, gap, stop rule
    double* obj = scal + kFistaHistory;
    const double cur = 0.5 * tot[2] + gamma * tot[0];
    obj[2 * it] = cur;
    obj[2 * it + 1] = gamma * tot[1];
    int crit = kTvRunning;
    if (it >= 1) {
      const double prev = obj[2 * (it - 1)];
      if (fabs(cur - prev) < tol * fabs(cur) || (cur == 0 && prev == 0 && tol > 0)) crit = kTvRtol;
      if (it >= maxit) crit = kTvMaxit;
    }
    if (crit != kTvRunning) {
      scal[2] = double(it);
      scal[1] = double(crit);
    }
    scal[0] = tn;
  });
}

// z = x - gamma D u: the step kernel's non-first form on the rectangular D.  That form also reads
// u at the output row (times beta = 0), so u has max(n, ne) rows.
template <typename T>
int tv_primal(int64_t n, int64_t d_nnz, const int32_t* d_indptr, const int32_t* d_indices,
              const T* d_data, const T* x, int nsig, double gamma, const T* u, T* z,
              cudaStream_t st) {
  Step<T> s{d_nnz, d_indptr, d_indices, d_data};
  s.x_cur = u;
  s.x_old = x;
  s.x_new = z;
  s.nsig = nsig;
  s.first = false;
  s.alpha = -gamma;
  s.beta = 0.0;
  s.gamma = 1.0;
  return run_step<T>(s, 0, n, nullptr, nullptr, st);
}

struct TvEdges {
  int64_t n, ne, ur;          // vertices, edges, rows of a U2 block (max(n, ne))
  int nsig;
  const int32_t* dt_indptr;
  const int32_t* dt_indices;
  double gamma, tau, tol;
  int maxit, cap;
};

template <typename T>
int tv_edges(const TvEdges& p, const T* dt_data, const T* wv, const T* x, const T* z, T* U2, T* G,
             int it, double* scal, cudaStream_t st) {
  const Lanes lanes = fista_lanes(p.nsig);
  const int64_t blk = p.ur * p.nsig;
  const int blocks = pass_blocks(std::max(p.ne, p.n), kThreads / lanes.w, kFistaMaxBlocks);
  return launch_lanes(lanes, [&](auto V) {
    tv_edge_kernel<T, decltype(V)::value><<<blocks, kThreads, 0, st>>>(
        p.n, p.ne, p.nsig, lanes.w, p.dt_indptr, p.dt_indices, dt_data, wv, x, z,
        U2 + (it % 2) * blk, U2 + ((it + 1) % 2) * blk, G, p.gamma, p.tau, p.tol, it, p.maxit, scal);
    GSP_LAUNCH_CHECK("tv_edge_kernel");
    return GSP_OK;
  });
}

static int tv_check(const TvEdges& p, int it0, int it1) {
  GSP_REQUIRE(p.n >= 1 && p.ne >= 1 && p.nsig >= 1, "prox_tv: empty problem");
  GSP_REQUIRE(p.gamma > 0 && p.tau > 0 && p.tol >= 0, "prox_tv: gamma, tau > 0 and tol >= 0");
  GSP_REQUIRE(p.maxit >= 1, "prox_tv: maxit >= 1");
  GSP_REQUIRE(it0 >= 0 && it0 <= it1 && it1 <= p.cap, "bad iteration range");
  return GSP_OK;
}

template <typename T>
int prox_tv_run(const TvEdges& p, int64_t d_nnz, const int32_t* d_indptr,
                const int32_t* d_indices, const T* d_data, const T* dt_data, const T* x, T* z,
                T* U2, T* G, int it0, int it1, double* scal, cudaStream_t st) {
  int rc = tv_check(p, it0, it1);
  if (rc != GSP_OK) return rc;
  const int64_t blk = p.ur * p.nsig;
  for (int it = it0; it < it1; ++it) {
    rc = tv_primal<T>(p.n, d_nnz, d_indptr, d_indices, d_data, x, p.nsig, p.gamma,
                      U2 + (it % 2) * blk, z, st);
    if (rc != GSP_OK) return rc;
    rc = tv_edges<T>(p, dt_data, z, x, z, U2, G, it, scal, st);
    if (rc != GSP_OK) return rc;
  }
  return GSP_OK;
}

}  // namespace gsp

extern "C" {
#define GSP_PROX_TV_API(SUF, T)                                                                    \
  int gsp_prox_tv_##SUF(int64_t n, int64_t n_edges, int64_t d_nnz, const int32_t* d_indptr,       \
                        const int32_t* d_indices, const T* d_data, const int32_t* dt_indptr,      \
                        const int32_t* dt_indices, const T* dt_data, const T* x, int64_t nsig,    \
                        double gamma, double tau, double tol, int maxit, T* z, T* U2, T* G,       \
                        int it0, int it1, int cap, double* scal_dev, void* stream) {              \
    GSP_REQUIRE(nsig >= 1 && nsig < (int64_t(1) << 31), "nsig out of range");                    \
    const gsp::TvEdges p{n, n_edges, std::max(n, n_edges), (int)nsig, dt_indptr, dt_indices,      \
                         gamma, tau, tol, maxit, cap};                                            \
    return gsp::prox_tv_run<T>(p, d_nnz, d_indptr, d_indices, d_data, dt_data, x, z, U2, G, it0,  \
                               it1, scal_dev, gsp::as_stream(stream));                            \
  }                                                                                                \
  int gsp_prox_tv_edges_##SUF(int64_t n, int64_t n_edges, const int32_t* dt_indptr,               \
                              const int32_t* dt_indices, const T* dt_data, const T* w,            \
                              const T* x, const T* z, int64_t nsig, double gamma, double tau,     \
                              double tol, int maxit, T* U2, T* G, int it, int cap,                \
                              double* scal_dev, void* stream) {                                   \
    GSP_REQUIRE(nsig >= 1 && nsig < (int64_t(1) << 31), "nsig out of range");                    \
    const gsp::TvEdges p{n, n_edges, std::max(n, n_edges), (int)nsig, dt_indptr, dt_indices,      \
                         gamma, tau, tol, maxit, cap};                                            \
    int rc = gsp::tv_check(p, it, it + 1);                                                        \
    if (rc != GSP_OK) return rc;                                                                  \
    return gsp::tv_edges<T>(p, dt_data, w, x, z, U2, G, it, scal_dev, gsp::as_stream(stream));    \
  }                                                                                                \
  int gsp_prox_tv_primal_##SUF(int64_t n, int64_t d_nnz, const int32_t* d_indptr,                 \
                               const int32_t* d_indices, const T* d_data, const T* x,             \
                               int64_t nsig, double gamma, const T* u, T* z, void* stream) {      \
    GSP_REQUIRE(n >= 1 && nsig >= 1 && nsig < (int64_t(1) << 31), "bad sizes");                  \
    return gsp::tv_primal<T>(n, d_nnz, d_indptr, d_indices, d_data, x, (int)nsig, gamma, u, z,    \
                             gsp::as_stream(stream));                                             \
  }
GSP_PROX_TV_API(f32, float)
GSP_PROX_TV_API(f64, double)
}
