// Accelerated forward-backward (FISTA) for simplex-constrained Tikhonov classification.
//
// Replaces pyunlocbox.solvers.forward_backward + solve on the problem of
// pygsp/learning.py:42-180 (classification_tikhonov_simplex):
//   min_X  tau tr(X^T L X) + ||M (X - Y)||^2   s.t. every row of X on the probability simplex,
// where the reference runs, per iteration, one SciPy SpMM for the gradient, a second one for the
// objective (smooth_eval, :160-164) and a Python loop over the vertices for the projection
// (proj_simplex, :121-158).  Here an iteration is two launches:
//
//   spmm  LX_k = L X_k                                   (cheby_step, FIRST form, alpha = 1)
//   row   partial sums of x_k'(L x_k), ||M(x_k - Y)||^2, ||x_k - x_{k-1}||^2 ;
//         y = x_k + beta (x_k - x_{k-1}),  L y = (1 + beta) L x_k - beta L x_{k-1}  (no 2nd SpMM)
//         x_{k+1} = proj_simplex(y - step * 2 (M (y - Y) + tau L y))  over x_{k-1}
//         the last block to finish reduces the partials in block order and applies the stop
//         tests of pyunlocbox.solvers.solve to x_k.
//
// Once a test has fired every later row launch returns at once, so the buffer of the stopping
// iterate is never written again: with X2 = [B0 | B1], iterate k lives in B[k % 2].
// The one-hot Y is never formed: label[row] is the class of a labelled vertex, -1 otherwise.
// The scratch has the FISTA layout of csrc/reduce.cuh; its history holds the objective of
// iterate k at k.
#include <math.h>

#include "reduce.cuh"
#include "step.cuh"

namespace gsp {

constexpr int kFbMaxClasses = 256;

enum { kCritNone = 0, kCritAtol = 1, kCritDtol = 2, kCritRtol = 3, kCritXtol = 4, kCritMaxit = 5 };

struct FbStop {
  double atol, dtol, rtol, xtol;   // NaN = off (every comparison with NaN is false)
  int maxit;                       // < 0 = off
};

template <typename T>
__global__ void __launch_bounds__(kThreads)
fb_init_kernel(int64_t n, int C, const int32_t* __restrict__ label, T* __restrict__ X0,
               double* scal) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    scal[0] = 1.0;
    scal[1] = 0.0;
    scal[2] = 0.0;
    reinterpret_cast<unsigned long long*>(scal)[3] = 0ull;
  }
  const int64_t total = n * C;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int64_t row = i / C;
    X0[i] = T(label[row] == int(i - row * C) ? 1 : 0);
  }
}

// One iteration (k = it): see the file comment.  V values per lane: V == 1 runs a sub-warp of
// w = 2^ceil(log2 C) lanes per row (32 / w rows per warp); V > 1 a warp per row (w = 32).
// Xprev may alias Xout (every element is read before the same thread overwrites it).
template <typename T, int V>
__global__ void __launch_bounds__(kThreads)
fb_row_kernel(int64_t n, int C, int w, const int32_t* __restrict__ label,
              const T* __restrict__ Xk, const T* Xprev, const T* __restrict__ LXk,
              const T* __restrict__ LXprev, T* Xout, double tau, double step, int it, FbStop stop,
              double* scal) {
  if (scal[1] != 0.0) return;                      // stopped at an earlier iteration
  const double t = scal[0];
  const double tn = (1.0 + sqrt(1.0 + 4.0 * t * t)) / 2.0;
  const double beta = (t - 1.0) / tn;
  const int lane = threadIdx.x % w, g = threadIdx.x / w, rpb = kThreads / w;
  double a_lap = 0, a_fit = 0, a_dx = 0;
  for (int64_t r0 = int64_t(blockIdx.x) * rpb; r0 < n; r0 += int64_t(gridDim.x) * rpb) {
    const int64_t row = r0 + g;                    // r0 is block-uniform: every lane iterates
    const bool valid = row < n;
    const int lab = valid ? label[row] : -1;
    double u[V];
    unsigned act = 0;
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int c = lane + v * w;
      u[v] = 0;
      if (valid && c < C) {
        const int64_t i = row * C + c;
        const double xk = double(Xk[i]), xp = double(Xprev[i]);
        const double lx = double(LXk[i]), lxp = double(LXprev[i]);
        a_lap += xk * lx;
        a_dx += (xk - xp) * (xk - xp);
        const double yv = c == lab ? 1.0 : 0.0;
        double fit = 0;
        const double y = xk + beta * (xk - xp);
        if (lab >= 0) {
          a_fit += (xk - yv) * (xk - yv);
          fit = y - yv;
        }
        const double ly = (1.0 + beta) * lx - beta * lxp;
        u[v] = y - step * (2.0 * (fit + tau * ly));
        act |= 1u << v;
      }
    }
    // Michelot: theta = (sum of the active values - 1) / their number; drop the values <= theta;
    // repeat until the active set is stable.  It only shrinks and always keeps the largest value,
    // so it ends after at most C rounds.  The loop is warp-uniform (the shuffles need every lane).
    double theta = 0;
    for (;;) {
      double s = 0;
      int cnt = 0;
#pragma unroll
      for (int v = 0; v < V; ++v)
        if (act >> v & 1u) { s += u[v]; ++cnt; }
      s = group_sum(s, w);
      cnt = group_sum(cnt, w);
      theta = (s - 1.0) / double(cnt > 0 ? cnt : 1);
      unsigned keep = 0;
#pragma unroll
      for (int v = 0; v < V; ++v)
        if ((act >> v & 1u) && u[v] > theta) keep |= 1u << v;
      const bool changed = keep != act;
      act = keep;
      if (!__any_sync(0xffffffffu, changed)) break;
    }
#pragma unroll
    for (int v = 0; v < V; ++v) {
      const int c = lane + v * w;
      if (valid && c < C) Xout[row * C + c] = T(fmax(u[v] - theta, 0.0));
    }
  }

  const double sums[3] = {a_lap, a_fit, a_dx};
  fista_last_block(sums, scal, [&](const double (&tot)[3]) {   // objective, stop rule
    double* obj = scal + kFistaHistory;
    const double cur = tau * tot[0] + tot[1];
    obj[it] = cur;
    int crit = kCritNone;
    if (it >= 1) {
      const double prev = obj[it - 1];
      if (cur < stop.atol) crit = kCritAtol;
      if (fabs(cur - prev) < stop.dtol) crit = kCritDtol;
      double div = cur;
      if (div == 0) div = prev != 0 ? prev : 1.0;
      if (fabs((cur - prev) / div) < stop.rtol) crit = kCritRtol;
      if (sqrt(tot[2]) / sqrt(double(n) * double(C)) < stop.xtol) crit = kCritXtol;
      if (stop.maxit >= 0 && it >= stop.maxit) crit = kCritMaxit;
    }
    if (crit != kCritNone) {
      scal[2] = double(it);
      scal[1] = double(crit);
    }
    scal[0] = tn;
  });
}

template <typename T>
int fb_simplex_run(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                   const T* data, const int32_t* label, int64_t nclass, double tau, double step,
                   const double* tol, int maxit, T* X2, T* LX2, int it0, int it1, int cap,
                   double* scal, const gsp_tile_plan* plan, cudaStream_t st) {
  GSP_REQUIRE(n >= 1 && nclass >= 1 && nclass <= kFbMaxClasses,
              "simplex classification: 1..256 classes");
  const int C = (int)nclass;
  GSP_REQUIRE(it0 >= 0 && it0 <= it1 && it1 <= cap, "bad iteration range");
  GSP_REQUIRE(tau > 0 && step > 0, "tau and step must be positive");
  GSP_REQUIRE(tol != nullptr, "tol_host is required");
  const FbStop stop{tol[0], tol[1], tol[2], tol[3], maxit};
  const Lanes lanes = fista_lanes(C);               // V <= 8 for C <= 256: one chunk of columns
  const int blocks = pass_blocks(n, kThreads / lanes.w, kFistaMaxBlocks);
  const int64_t nc = n * C;
  if (it0 == 0) {
    const int ib = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(nc, kThreads),
                                                                 int64_t(sm_count()) * 8));
    fb_init_kernel<T><<<ib, kThreads, 0, st>>>(n, C, label, X2, scal);
    GSP_LAUNCH_CHECK("fb_init_kernel");
  }
  Step<T> lap{nnz, indptr, indices, data};        // L X_k: the first form, alpha = 1, no r_i
  lap.r_rows = n;
  lap.nsig = C;
  lap.first = true;
  lap.alpha = 1.0;
  for (int it = it0; it < it1; ++it) {
    T* Xk = X2 + (it % 2) * nc;
    T* Xo = X2 + ((it + 1) % 2) * nc;
    T* LXk = LX2 + (it % 2) * nc;
    T* LXo = LX2 + ((it + 1) % 2) * nc;
    // iteration 0 has no x_{-1}: read x_0 in its place (beta = 0 there)
    const T* Xp = it == 0 ? Xk : Xo;
    const T* LXp = it == 0 ? LXk : LXo;
    lap.x_cur = lap.x_old = Xk;
    lap.x_new = lap.r = LXk;
    int rc = run_step<T>(lap, 0, n, plan, nullptr, st);
    if (rc != GSP_OK) return rc;
    rc = launch_lanes(lanes, [&](auto V) {
      fb_row_kernel<T, decltype(V)::value><<<blocks, kThreads, 0, st>>>(
          n, C, lanes.w, label, Xk, Xp, LXk, LXp, Xo, tau, step, it, stop, scal);
      GSP_LAUNCH_CHECK("fb_row_kernel");
      return GSP_OK;
    });
    if (rc != GSP_OK) return rc;
  }
  return GSP_OK;
}

}  // namespace gsp

extern "C" {
#define GSP_FB_SIMPLEX_API(SUF, T)                                                                \
  int gsp_fb_simplex_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices, \
                           const T* data, const int32_t* label, int64_t nclass, double tau,       \
                           double step, const double* tol_host, int maxit, T* X2, T* LX2,         \
                           int it0, int it1, int cap, double* scal_dev,                           \
                           const gsp_tile_plan* plan_host, void* stream) {                        \
    return gsp::fb_simplex_run<T>(n, nnz, indptr, indices, data, label, nclass, tau, step,        \
                                  tol_host, maxit, X2, LX2, it0, it1, cap, scal_dev, plan_host,   \
                                  gsp::as_stream(stream));                                        \
  }
GSP_FB_SIMPLEX_API(f32, float)
GSP_FB_SIMPLEX_API(f64, double)
}
