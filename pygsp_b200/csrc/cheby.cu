// Chebyshev recurrence on a CSR Laplacian -- the hot path.
//
// Replaces, for the path pygsp/filters/approximations.py:58-114 (cheby_op):
//   * scipy.sparse._sparsetools.csr_matvecs   (approximations.py:99,107)
//   * the dense "- twf_old" temporary          (approximations.py:107)
//   * the fancy-indexed r[tmpN + N*i] += c*T   (approximations.py:108-109)
// by ONE fused kernel per recurrence step:
//   x_new = alpha * (L x_cur) + beta * x_cur + gamma * x_old
//   r_i   = (first ? c_i0/2 * x_cur : r_i) + c_ik * x_new         i < nscales
// with alpha = 4/lmax, beta = -2, gamma = -1 (first step: 2/lmax, -1, 0), so
// the CSR of L is used as stored (the reference builds a second scaled matrix
// "factor", approximations.py:105) and T_{k-2}/T_{k-1}/T_k make exactly one
// trip each through HBM per step.
//
// Layout: signals are (N, nsig) row-major (a vertex's nsig values adjacent),
// r is (nscales, N, nsig) -- the reference's filter-major (Nscales*N, Nsig).
//
// Lane mapping ("row group" kernel): G = 2^g lanes own one row, each lane a
// VEC-wide packet (16 B) of the row's columns.  The group loads G CSR entries
// with one coalesced access and broadcasts them with shuffles; every lane then
// gathers its packet of x_cur[col] -- a 16*G-byte contiguous, fully coalesced
// request per neighbour -- and accumulates in registers.  The accumulation
// order is the stored CSR order, i.e. the order scipy uses.
#include "step.cuh"

namespace gsp {

constexpr int kStepThreads = 256;

template <typename T>
struct StepCoef {
  T alpha, beta, gamma;
  T half_c0[kMaxScales];   // c[i,0]/2 (first step only)
  T ck[kMaxScales];        // c[i,k]
  // Clenshaw form: `r` holds nscales read-only source blocks s_i and the step is
  // x_new += sum_i ck[i] * s_i; nothing is accumulated into r.
  int add_source;
};

template <typename T, int VEC, int G, bool FIRST, bool SPMM>
__global__ void __launch_bounds__(kStepThreads)
cheby_step_rowgroup(int64_t row_begin, int64_t row_end,
                    const int32_t* __restrict__ indptr,
                    const int32_t* __restrict__ indices,
                    const T* __restrict__ vals,
                    const T* __restrict__ x_cur,   // rows referenced by indices
                    const T* x_old,                // may alias x_new (row-local)
                    T* x_new,
                    T* __restrict__ r,             // (nscales, r_rows, nsig)
                    int64_t r_rows, int nsig, int nscales,
                    StepCoef<T> coef, const int64_t* __restrict__ out_perm) {
  const int lane = threadIdx.x & (G - 1);
  const int64_t group = (int64_t(blockIdx.x) * kStepThreads + threadIdx.x) / G;
  const int64_t row = row_begin + group;
  // all lanes of a group share `row`; groups never straddle a warp (G <= 32)
  if (row >= row_end) return;
  const unsigned lane_in_warp = threadIdx.x & 31;
  const unsigned gmask = (G == 32) ? 0xffffffffu
                                   : (((1u << G) - 1u) << (lane_in_warp & ~(G - 1)));

  const int start = __ldg(indptr + row);
  const int end = __ldg(indptr + row + 1);
  const int64_t out_row = out_perm ? __ldg(out_perm + row) : row;   // x_new only

  // every lane of the group runs the same trip count (the shuffles below need
  // the whole group); lanes past the last column are merely predicated off
  for (int cbase = 0; cbase < nsig; cbase += G * VEC) {
    const int c0 = cbase + lane * VEC;
    const bool active = c0 < nsig;
    Vec<T, VEC> acc, xo, xc;
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc.v[v] = xo.v[v] = xc.v[v] = T(0);

    // streaming operands first: they are in flight while the gather runs.  x_cur's own row is
    // read only when a term uses it, so a plain product (FIRST, beta = 0, no accumulator)
    // indexes x_cur by column alone and the matrix may be rectangular (gsp_spmm_*)
    if (active) {
      if (!FIRST) xo = load_vec_stream<T, VEC>(x_old + row * nsig + c0);
      if (!FIRST || coef.beta != T(0) || nscales > 0)
        xc = load_vec_ro<T, VEC>(x_cur + row * nsig + c0);
    }

    if (SPMM) {
      for (int base = start; base < end; base += G) {
        const int mine = base + lane;
        int col = 0;
        T val = T(0);
        if (mine < end) {
          col = __ldg(indices + mine);
          val = __ldg(vals + mine);
        }
        const int cnt = min(G, end - base);
#pragma unroll 4
        for (int j = 0; j < cnt; ++j) {
          const int cj = __shfl_sync(gmask, col, j, G);
          const T vj = __shfl_sync(gmask, val, j, G);
          if (active) {
            const Vec<T, VEC> xn = load_vec_ro<T, VEC>(x_cur + int64_t(cj) * nsig + c0);
#pragma unroll
            for (int v = 0; v < VEC; ++v) acc.v[v] = fma(vj, xn.v[v], acc.v[v]);
          }
        }
      }
    }
    if (!active) continue;

    Vec<T, VEC> xn;
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
      T t = fma(coef.alpha, acc.v[v], coef.beta * xc.v[v]);
      if (!FIRST) t = fma(coef.gamma, xo.v[v], t);
      xn.v[v] = t;
    }
    if (coef.add_source) {
      for (int i = 0; i < nscales; ++i) {
        const Vec<T, VEC> sv =
            load_vec_stream<T, VEC>(r + (int64_t(i) * r_rows + row) * nsig + c0);
#pragma unroll
        for (int v = 0; v < VEC; ++v) xn.v[v] = fma(coef.ck[i], sv.v[v], xn.v[v]);
      }
      store_vec_stream<T, VEC>(x_new + out_row * nsig + c0, xn);
      continue;
    }
    store_vec_stream<T, VEC>(x_new + out_row * nsig + c0, xn);

    for (int i = 0; i < nscales; ++i) {
      T* rp = r + (int64_t(i) * r_rows + row) * nsig + c0;
      Vec<T, VEC> rv;
      if (FIRST) {
#pragma unroll
        for (int v = 0; v < VEC; ++v)
          rv.v[v] = fma(coef.ck[i], xn.v[v], coef.half_c0[i] * xc.v[v]);
      } else {
        rv = load_vec_stream<T, VEC>(rp);
#pragma unroll
        for (int v = 0; v < VEC; ++v) rv.v[v] = fma(coef.ck[i], xn.v[v], rv.v[v]);
      }
      store_vec_stream<T, VEC>(rp, rv);
    }
  }
}

// r_i += c_ik * x   for filter banks wider than kMaxScales (no SpMM)
template <typename T>
__global__ void cheby_axpy_scales(int64_t count, const T* __restrict__ x,
                                  T* __restrict__ r, int64_t r_stride, int nscales,
                                  StepCoef<T> coef, bool first,
                                  const T* __restrict__ x0) {
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (; i < count; i += stride) {
    const T xv = x[i];
    for (int s = 0; s < nscales; ++s) {
      T* rp = r + int64_t(s) * r_stride + i;
      *rp = first ? fma(coef.ck[s], xv, coef.half_c0[s] * x0[i]) : fma(coef.ck[s], xv, *rp);
    }
  }
}

template <typename T, int VEC, int G>
static int launch_group(bool first, bool spmm, int64_t row_begin, int64_t row_end,
                        const int32_t* indptr, const int32_t* indices, const T* vals,
                        const T* x_cur, const T* x_old, T* x_new, T* r, int64_t r_rows,
                        int nsig, int nscales, const StepCoef<T>& coef, cudaStream_t st,
                        const int64_t* out_perm) {
  const int64_t rows = row_end - row_begin;
  if (rows <= 0) return GSP_OK;
  const int64_t blocks = ceil_div(rows * G, kStepThreads);
  GSP_REQUIRE(blocks < (int64_t(1) << 31), "row range too large for one launch");
  dim3 grid((unsigned)blocks), block(kStepThreads);
#define GSP_GO(F, S)                                                                   \
  cheby_step_rowgroup<T, VEC, G, F, S><<<grid, block, 0, st>>>(                        \
      row_begin, row_end, indptr, indices, vals, x_cur, x_old, x_new, r, r_rows, nsig, \
      nscales, coef, out_perm)
  if (first && spmm) GSP_GO(true, true);
  else if (first) GSP_GO(true, false);
  else if (spmm) GSP_GO(false, true);
  else GSP_GO(false, false);
#undef GSP_GO
  GSP_LAUNCH_CHECK("cheby_step_rowgroup");
  return GSP_OK;
}

template <typename T, int VEC>
static int launch_vec(int groups_needed, bool first, bool spmm, int64_t rb, int64_t re,
                      const int32_t* indptr, const int32_t* indices, const T* vals,
                      const T* x_cur, const T* x_old, T* x_new, T* r, int64_t r_rows,
                      int nsig, int nscales, const StepCoef<T>& coef, cudaStream_t st,
                      const int64_t* out_perm) {
#define GSP_CASE(GG)                                                                     \
  return launch_group<T, VEC, GG>(first, spmm, rb, re, indptr, indices, vals, x_cur,     \
                                  x_old, x_new, r, r_rows, nsig, nscales, coef, st, out_perm)
  if (groups_needed <= 1) GSP_CASE(1);
  if (groups_needed <= 2) GSP_CASE(2);
  if (groups_needed <= 4) GSP_CASE(4);
  if (groups_needed <= 8) GSP_CASE(8);
  if (groups_needed <= 16) GSP_CASE(16);
  GSP_CASE(32);
#undef GSP_CASE
}

template <typename T> struct MaxVec;
template <> struct MaxVec<float> { static constexpr int value = 4; };
template <> struct MaxVec<double> { static constexpr int value = 2; };


template <typename T>
int cheby_step(const Step<T>& s, int64_t rb, int64_t re, cudaStream_t st) {
  constexpr int MV = MaxVec<T>::value;
  const int nsig = s.nsig;
  const bool vec_ok = (nsig % MV == 0) && aligned16(s.x_cur) && aligned16(s.x_new) &&
                      aligned16(s.r) && (s.first || aligned16(s.x_old));
  for (int s0 = 0; s0 < s.nscales || s0 == 0; s0 += kMaxScales) {
    const int ns = min(kMaxScales, s.nscales - s0);
    StepCoef<T> coef;
    coef.alpha = T(s.alpha);
    coef.beta = T(s.beta);
    coef.gamma = T(s.gamma);
    coef.add_source = s.add_source ? 1 : 0;
    for (int i = 0; i < kMaxScales; ++i) {
      coef.ck[i] = i < ns ? T(s.ck[s0 + i]) : T(0);
      coef.half_c0[i] = (s.first && i < ns) ? T(0.5 * s.c0[s0 + i]) : T(0);
    }
    T* rs = s.r + int64_t(s0) * s.r_rows * nsig;
    if (s0 == 0) {
      int rc;
      if (vec_ok)
        rc = launch_vec<T, MV>((nsig + MV - 1) / MV, s.first, true, rb, re, s.indptr, s.indices,
                               s.vals, s.x_cur, s.x_old, s.x_new, rs, s.r_rows, nsig, ns, coef, st,
                               s.out_perm);
      else
        rc = launch_vec<T, 1>(nsig, s.first, true, rb, re, s.indptr, s.indices, s.vals, s.x_cur,
                              s.x_old, s.x_new, rs, s.r_rows, nsig, ns, coef, st, s.out_perm);
      if (rc != GSP_OK) return rc;
    } else {
      // remaining scales of a wide bank: r_i (+)= c_ik * x_new, no second SpMM
      const int64_t count = (re - rb) * nsig;
      if (count > 0) {
        const int blocks = (int)std::min<int64_t>(ceil_div(count, 256), int64_t(sm_count()) * 16);
        cheby_axpy_scales<T><<<blocks, 256, 0, st>>>(
            count, s.x_new + rb * nsig, rs + rb * nsig, s.r_rows * nsig, ns, coef, s.first,
            s.x_cur + rb * nsig);
        GSP_LAUNCH_CHECK("cheby_axpy_scales");
      }
    }
    if (s.nscales == 0) break;
  }
  return GSP_OK;
}

template <typename T>
int run_step(const Step<T>& s, int64_t rb, int64_t re, const gsp_tile_plan* plan,
             const gsp_halo_fusion* halo, cudaStream_t st) {
  const bool tiled = tiled_step_applies(s, rb, plan);
  if (halo && !tiled)
    return fail(GSP_ERR_UNSUPPORTED, "fused halo step: the tiled kernel does not apply (it needs "
                "a tile plan, at most 16 filters and 16-byte aligned blocks)");
  int64_t done = 0;
  if constexpr (std::is_same<T, float>::value) {
    if (halo) {
      // (1) The boundary ("front") tiles -- those holding rows that read halo columns or that some
      // neighbour needs -- with the halo-capable instantiation: wait for the neighbours' flags,
      // coherent gathers, peer stores of the new boundary rows, publish.  (2) The interior tiles
      // with the plain instantiation.  One kernel for both is slower per step (DESIGN.md section
      // 5): under the 60-register cap ptxas spills the boundary code's state inside the interior
      // gather loop.  The front launch is a few dozen tiles and publishes before the interior
      // tiles run, so the neighbours' next front launch finds the flag set.
      GSP_REQUIRE(rb == 0, "fused halo step needs the whole row block");
      const int64_t R = plan->rows_per_tile;
      const int64_t front = ceil_div(std::max<int64_t>(halo->publish ? halo->n_push_rows : 0,
                                                       halo->n_boundary_rows), R) * R;
      GSP_REQUIRE(front <= (re / R) * R, "boundary rows must lie inside the full tiles");
      if (front > 0) {
        Step<float> fs = s;
        fs.reverse = false;
        int rc = cheby_step_tiled_f32(fs, 0, front, *plan, halo, &done, st);
        if (rc != GSP_OK) return rc;
        GSP_REQUIRE(done == front, "front tiles must be whole tiles");
      }
    }
    if (tiled) {
      int64_t interior = 0;
      int rc = cheby_step_tiled_f32(s, rb + done, re, *plan, nullptr, &interior, st);
      if (rc != GSP_OK) return rc;
      done += interior;
    }
  }
  // the < rows_per_tile remainder (interior rows by the fused-step condition), or every row
  return cheby_step<T>(s, rb + done, re, st);
}

// Full operator (approximations.py:58-114): K = m-1 fused steps on `stream`.
template <typename T>
int cheby_op(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
             const T* vals, double lmax, const double* coeffs, int nscales, int m, const T* x,
             int nsig, T* r, T* work, const gsp_tile_plan* plan, cudaStream_t st) {
  GSP_REQUIRE(n >= 0 && nsig >= 1 && nscales >= 1, "bad sizes");
  GSP_REQUIRE(m >= 2, "The coefficients have an invalid shape");   // approximations.py:83-84
  GSP_REQUIRE(lmax > 0 && lmax == lmax, "lmax must be positive");
  if (n == 0) return GSP_OK;
  double ck[1024], c0[1024];
  GSP_REQUIRE(nscales <= 1024, "at most 1024 filters per call");
  T* buf[2] = {work, work + n * int64_t(nsig)};
  Step<T> s{nnz, indptr, indices, vals};
  s.r = r;
  s.r_rows = n;
  s.nsig = nsig;
  const T* t_old = x;
  const T* t_cur = x;
  for (int k = 1; k < m; ++k) {
    forward_coefs(s, k, m, nscales, lmax, coeffs, ck, c0);
    // T_1 into buf[0]; T_k written over T_{k-2} (row-local) except for k == 2, where T_0 is the
    // caller's input
    T* dst = k == 1 ? buf[0] : (k == 2 ? buf[1] : const_cast<T*>(t_old));
    s.x_cur = t_cur;
    s.x_old = k == 1 ? nullptr : t_old;
    s.x_new = dst;
    int rc = run_step<T>(s, 0, n, plan, nullptr, st);
    if (rc != GSP_OK) return rc;
    t_old = t_cur;
    t_cur = dst;
  }
  return GSP_OK;
}

// out = sum_i w[i] * src_i   (src: (nsrc, count) blocks) -- the top Clenshaw term S_K
template <typename T>
__global__ void combine_sources(int64_t count, const T* __restrict__ src, int nsrc,
                                StepCoef<T> coef, T* __restrict__ out) {
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (; i < count; i += stride) {
    T acc = T(0);
    for (int s = 0; s < nsrc; ++s) acc = fma(coef.ck[s], src[int64_t(s) * count + i], acc);
    out[i] = acc;
  }
}

// Chebyshev sums by Clenshaw's recurrence (SURVEY.md 8f ranks 1 and 2).  For source
// blocks s_i (nsrc of them, (nsrc, n, nsig) in memory) and coefficient rows c_i:
//   out = sum_i p_i(L) s_i,   p_i = c_i0/2 + sum_k c_ik T_k(Lt),  Lt = (2/lmax) L - I
// is evaluated as ONE backward recurrence on an (n, nsig) block,
//   S_k = sum_i c_ik s_i ;  b_k = S_k + 2 Lt b_{k+1} - b_{k+2} ;  out = S_0/2 + Lt b_1 - b_2,
// i.e. K SpMMs in total -- the reference's synthesis (filter.py:313-322) runs nsrc
// separate forward recurrences, nsrc*K SpMMs -- and no accumulator block.  With
// nsrc = 1 this is the single-filter Clenshaw evaluation (b_K = c_K x is folded into
// the first step).  work holds 2*n*nsig elements.  Rounding differs from the forward
// recurrence, the value does not (tests: same tolerance against the float64 oracle).
//
// With `pairs` (float32, one source, a tile plan; work then holds 3*n*nsig elements) the middle
// steps k = K-3 .. 1 run two per launch (cheby_pair_tiled, csrc/cheby_tiled.cu): b_k goes to the
// free third block, b_{k-1} over b_{k+2}, and the block of b_{k+1} becomes the free one.  The
// first two steps, the last one and a left-over middle step are single launches.  Rows past the
// last full tile take the row-group kernel: step A on them before the paired launch (it reads
// only blocks complete by then, and the launch's B tiles gather its rows), step B after it.
struct ClenshawPairs {
  const int32_t* slots_fwd;
  const int32_t* slots_rev;
  const int32_t* nbr_ptr;
  const int32_t* nbr_idx;
  unsigned* tile_done;
};

template <typename T>
int cheby_clenshaw(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                   const T* vals, double lmax, const double* c, int nsrc, int m, const T* src,
                   int nsig, T* out, T* work, const gsp_tile_plan* plan, cudaStream_t st,
                   const ClenshawPairs* pairs = nullptr, const gsp_ring_plan* ring = nullptr) {
  GSP_REQUIRE(n >= 0 && nsig >= 1 && nsrc >= 1 && nsrc <= kMaxScales, "bad sizes");
  GSP_REQUIRE(m >= 2, "The coefficients have an invalid shape");
  GSP_REQUIRE(lmax > 0 && lmax == lmax, "lmax must be positive");
  if (n == 0) return GSP_OK;
  const int K = m - 1;
  T* buf[2] = {work, work + n * int64_t(nsig)};
  double ck[kMaxScales];
  Step<T> s{nnz, indptr, indices, vals};
  s.r_rows = n;
  s.nsig = nsig;
  s.ring = ring;
  const T* b_cur = buf[0];
  const T* b_old = nullptr;
  int k_next;
  if (nsrc == 1) {
    // b_{K-1} from x (with K == 1: out)
    clenshaw_coefs(s, K - 1, m, 1, lmax, c, ck);
    s.x_cur = src;
    s.x_new = s.r = K == 1 ? out : buf[0];
    int rc = run_step<T>(s, 0, n, plan, nullptr, st);
    if (rc != GSP_OK || K == 1) return rc;
    k_next = K - 2;
  } else {
    // b_K = S_K by one combine pass
    StepCoef<T> coef;
    memset(&coef, 0, sizeof(coef));
    for (int i = 0; i < nsrc; ++i) coef.ck[i] = T(c[int64_t(i) * m + K]);
    const int64_t count = n * int64_t(nsig);
    const int blocks = (int)std::min<int64_t>(ceil_div(count, 256), int64_t(sm_count()) * 16);
    combine_sources<T><<<blocks, 256, 0, st>>>(count, src, nsrc, coef, buf[0]);
    GSP_LAUNCH_CHECK("combine_sources");
    k_next = K - 1;
  }
  s.r = const_cast<T*>(src);                      // read-only source blocks
  T* spare = pairs ? work + 2 * n * int64_t(nsig) : nullptr;   // the third block of a paired call
  unsigned launch_index = 0;
  for (int k = k_next; k >= 0; --k) {
    if constexpr (std::is_same<T, float>::value) {
      if (pairs && b_old && k >= 2) {
        double ck2[kMaxScales];
        Step<float> sa = s, sb = s;
        clenshaw_coefs(sa, k, m, 1, lmax, c, ck);
        clenshaw_coefs(sb, k - 1, m, 1, lmax, c, ck2);
        sa.x_cur = b_cur; sa.x_old = b_old; sa.x_new = spare;
        sb.x_cur = spare; sb.x_old = b_cur; sb.x_new = const_cast<float*>(b_old);
        const int64_t tiles = n / plan->rows_per_tile;
        if (launch_index == 0)
          GSP_CUDA(cudaMemsetAsync(pairs->tile_done, 0, tiles * sizeof(unsigned), st));
        const bool rev = (launch_index & 1) != 0;
        PairLaunch pl{&sb, rev ? pairs->slots_rev : pairs->slots_fwd, pairs->nbr_ptr,
                      pairs->nbr_idx, pairs->tile_done, ++launch_index};
        const int64_t tiled_rows = tiles * plan->rows_per_tile;
        int rc = cheby_step<float>(sa, tiled_rows, n, st);
        if (rc != GSP_OK) return rc;
        int64_t done = 0;
        rc = cheby_step_tiled_f32(sa, 0, n, *plan, nullptr, &done, st, &pl);
        if (rc != GSP_OK) return rc;
        GSP_REQUIRE(done == tiled_rows, "the paired launch covers the full tiles");
        rc = cheby_step<float>(sb, tiled_rows, n, st);
        if (rc != GSP_OK) return rc;
        float* freed = const_cast<float*>(b_cur);
        b_cur = sb.x_new;
        b_old = spare;
        spare = freed;
        --k;
        continue;
      }
    }
    clenshaw_coefs(s, k, m, nsrc, lmax, c, ck);
    T* dst = k == 0 ? out : (b_old ? const_cast<T*>(b_old) : buf[1]);
    s.x_cur = b_cur;
    s.x_old = b_old ? b_old : b_cur;              // no b_{k+2} yet: any valid block, times gamma = 0
    s.x_new = dst;
    int rc = run_step<T>(s, 0, n, plan, nullptr, st);
    if (rc != GSP_OK) return rc;
    b_old = b_cur;
    b_cur = dst;
  }
  return GSP_OK;
}

// y = A x for a block of vectors (no recurrence, no r): used by Lanczos and
// exposed for callers that only need the product (learning.py CG, "next").
template <typename T>
int spmm_plain(int64_t n, const int32_t* indptr, const int32_t* indices, const T* vals,
               const T* x, int nsig, T* y, cudaStream_t st) {
  // x_new = 1 * (A x) + 0 * x ; FIRST form with nscales = 0 touches no r
  Step<T> s{0, indptr, indices, vals};
  s.x_cur = x;
  s.x_new = s.r = y;
  s.r_rows = n;
  s.nsig = nsig;
  s.first = true;
  s.alpha = 1.0;
  return run_step<T>(s, 0, n, nullptr, nullptr, st);
}

// a step as the C ABI passes it (gsp_cheby_step_*, gsp_cheby_step_halo_f32)
template <typename T>
static Step<T> abi_step(int first, int64_t nnz, const int32_t* indptr, const int32_t* indices,
                        const T* data, const T* x_cur, const T* x_old, T* x_new, T* r,
                        int64_t r_rows, int64_t nsig, int nscales, const double* ck,
                        const double* c0, double alpha, double beta, double gamma) {
  Step<T> s{nnz, indptr, indices, data};
  s.x_cur = x_cur;
  s.x_old = x_old;
  s.x_new = x_new;
  s.r = r;
  s.r_rows = r_rows;
  s.nsig = (int)nsig;
  s.first = first != 0;
  s.alpha = alpha;
  s.beta = beta;
  s.gamma = gamma;
  s.nscales = nscales;
  s.ck = ck;
  s.c0 = c0;
  return s;
}

template int cheby_step<float>(const Step<float>&, int64_t, int64_t, cudaStream_t);
template int cheby_step<double>(const Step<double>&, int64_t, int64_t, cudaStream_t);
template int run_step<float>(const Step<float>&, int64_t, int64_t, const gsp_tile_plan*,
                             const gsp_halo_fusion*, cudaStream_t);
template int run_step<double>(const Step<double>&, int64_t, int64_t, const gsp_tile_plan*,
                              const gsp_halo_fusion*, cudaStream_t);

}  // namespace gsp

// ------------------------------- C ABI ------------------------------------
extern "C" {

#define GSP_CHEBY_API(SUF, T)                                                                     \
  int gsp_cheby_op_##SUF(int64_t n, int64_t nnz, const int32_t* indptr, const int32_t* indices,   \
                         const T* data, double lmax, const double* coeffs_host, int nscales,      \
                         int m, const T* x, int64_t nsig, T* r, T* work,                          \
                         const gsp_tile_plan* plan_host, void* stream) {                          \
    GSP_REQUIRE(nsig >= 1 && nsig <= (1 << 20), "nsig out of range");                             \
    return gsp::cheby_op<T>(n, nnz, indptr, indices, data, lmax, coeffs_host, nscales, m, x,      \
                            (int)nsig, r, work, plan_host, gsp::as_stream(stream));               \
  }                                                                                               \
  int gsp_cheby_step_##SUF(int first, int64_t row_begin, int64_t row_end, int64_t nnz,            \
                           const int32_t* indptr, const int32_t* indices, const T* data,          \
                           const T* x_cur, const T* x_old, T* x_new, T* r, int64_t r_rows,        \
                           int64_t nsig, int nscales, const double* ck_host,                      \
                           const double* c0_host, double alpha, double beta, double gamma,        \
                           const gsp_tile_plan* plan_host, void* stream) {                        \
    GSP_REQUIRE(nsig >= 1 && nsig <= (1 << 20), "nsig out of range");                             \
    return gsp::run_step<T>(gsp::abi_step<T>(first, nnz, indptr, indices, data, x_cur, x_old,      \
                                             x_new, r, r_rows, nsig, nscales, ck_host, c0_host,   \
                                             alpha, beta, gamma),                                 \
                            row_begin, row_end, plan_host, nullptr, gsp::as_stream(stream));      \
  }                                                                                               \
  int gsp_cheby_clenshaw_##SUF(int64_t n, int64_t nnz, const int32_t* indptr,                     \
                               const int32_t* indices, const T* data, double lmax,                \
                               const double* coeffs_host, int nsrc, int m, const T* sources,      \
                               int64_t nsig, T* out, T* work, const gsp_tile_plan* plan_host,     \
                               void* stream) {                                                    \
    GSP_REQUIRE(nsig >= 1 && nsig <= (1 << 20), "nsig out of range");                             \
    return gsp::cheby_clenshaw<T>(n, nnz, indptr, indices, data, lmax, coeffs_host, nsrc, m,      \
                                  sources, (int)nsig, out, work, plan_host,                       \
                                  gsp::as_stream(stream));                                        \
  }                                                                                               \
  int gsp_spmm_##SUF(int64_t n, const int32_t* indptr, const int32_t* indices, const T* data,     \
                     const T* x, int64_t nsig, T* y, void* stream) {                              \
    GSP_REQUIRE(nsig >= 1 && nsig <= (1 << 20), "nsig out of range");                             \
    return gsp::spmm_plain<T>(n, indptr, indices, data, x, (int)nsig, y, gsp::as_stream(stream)); \
  }

GSP_CHEBY_API(f32, float)
GSP_CHEBY_API(f64, double)

int gsp_cheby_clenshaw_pairs_wanted(int64_t n, int64_t nsig, const gsp_tile_plan* plan_host) {
  if (!plan_host || plan_host->rows_per_tile <= 0 || n / plan_host->rows_per_tile < 1) return 0;
  const char* d = getenv("GSPB200_TILE_VDIR");           // probe: vectors staged by TMA, no pairs
  if (d && *d && atoi(d) == 0) return 0;
  const char* v = getenv("GSPB200_CLENSHAW_PAIRS");      // A/B probe: 0 never, 1 whatever the size
  if (v && *v) return atoi(v) != 0;
  int dev = 0, l2 = 0;
  if (cudaGetDevice(&dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, dev) != cudaSuccess)
    return 0;
  return n * nsig * int64_t(sizeof(float)) > int64_t(l2);
}

int gsp_cheby_clenshaw_ring_f32(int64_t n, int64_t nnz, const int32_t* indptr,
                                const int32_t* indices, const float* data, double lmax,
                                const double* coeffs_host, int nsrc, int m, const float* sources,
                                int64_t nsig, float* out, float* work,
                                const gsp_tile_plan* plan_host, const gsp_ring_plan* ring_host,
                                const int32_t* slots_fwd, const int32_t* slots_rev,
                                const int32_t* nbr_ptr, const int32_t* nbr_idx,
                                uint32_t* tile_done, void* stream) {
  GSP_REQUIRE(nsig >= 1 && nsig <= (1 << 20), "nsig out of range");
  GSP_REQUIRE(!ring_host || (plan_host && ring_host->rows_per_tile == plan_host->rows_per_tile &&
                             ring_host->tile_meta && ring_host->runs && ring_host->local),
              "the ring plan must be one of the tile plan's rows per tile");
  if (!slots_fwd)
    return gsp::cheby_clenshaw<float>(n, nnz, indptr, indices, data, lmax, coeffs_host, nsrc, m,
                                      sources, (int)nsig, out, work, plan_host,
                                      gsp::as_stream(stream), nullptr, ring_host);
  GSP_REQUIRE(nsrc == 1, "paired steps take one source");
  GSP_REQUIRE(plan_host && plan_host->rows_per_tile > 0, "paired steps need a tile plan");
  GSP_REQUIRE(slots_fwd && slots_rev && nbr_ptr && nbr_idx && tile_done,
              "paired steps need a pair plan");
  gsp::Step<float> probe{nnz, indptr, indices, data};
  probe.x_cur = work;
  probe.x_old = work + n * nsig;
  probe.x_new = work + 2 * n * nsig;
  probe.r = const_cast<float*>(sources);
  probe.nscales = 1;
  GSP_REQUIRE(gsp::tiled_step_applies(probe, 0, plan_host) && gsp::aligned16(out),
              "paired steps need 16-byte aligned blocks");
  const gsp::ClenshawPairs pairs{slots_fwd, slots_rev, nbr_ptr, nbr_idx, tile_done};
  return gsp::cheby_clenshaw<float>(n, nnz, indptr, indices, data, lmax, coeffs_host, 1, m,
                                    sources, (int)nsig, out, work, plan_host,
                                    gsp::as_stream(stream), &pairs, ring_host);
}

int gsp_cheby_clenshaw_pairs_f32(int64_t n, int64_t nnz, const int32_t* indptr,
                                 const int32_t* indices, const float* data, double lmax,
                                 const double* coeffs_host, int m, const float* source,
                                 int64_t nsig, float* out, float* work,
                                 const gsp_tile_plan* plan_host, const int32_t* slots_fwd,
                                 const int32_t* slots_rev, const int32_t* nbr_ptr,
                                 const int32_t* nbr_idx, uint32_t* tile_done, void* stream) {
  GSP_REQUIRE(slots_fwd, "paired steps need a pair plan");
  return gsp_cheby_clenshaw_ring_f32(n, nnz, indptr, indices, data, lmax, coeffs_host, 1, m,
                                     source, nsig, out, work, plan_host, nullptr, slots_fwd,
                                     slots_rev, nbr_ptr, nbr_idx, tile_done, stream);
}

int gsp_cheby_step_halo_f32(int first, int64_t n_rows, int64_t nnz, const int32_t* indptr,
                            const int32_t* indices, const float* data, const float* x_cur,
                            const float* x_old, float* x_new, float* r, int64_t r_rows,
                            int64_t nsig, int nscales, const double* ck_host,
                            const double* c0_host, double alpha, double beta, double gamma,
                            int reverse, const gsp_tile_plan* plan_host,
                            const gsp_halo_fusion* halo_host, void* stream) {
  if (!halo_host) return gsp::fail(GSP_ERR_UNSUPPORTED, "fused halo step needs a halo description");
  GSP_REQUIRE(nscales <= gsp::kMaxScales, "too many filters for the fused step");
  gsp::Step<float> s = gsp::abi_step<float>(first, nnz, indptr, indices, data, x_cur, x_old, x_new,
                                            r, r_rows, nsig, nscales, ck_host, c0_host, alpha,
                                            beta, gamma);
  s.reverse = reverse != 0;
  return gsp::run_step<float>(s, 0, n_rows, plan_host, halo_host, gsp::as_stream(stream));
}

}  // extern "C"
