// One step of the Chebyshev recurrence (Step), its two back ends and the one dispatch between them.
//
//   cheby_step<T>          row-group kernel (csrc/cheby.cu): any dtype, width, row range, bank
//   cheby_step_tiled_f32   TMA-tiled kernel (csrc/cheby_tiled.cu): float32, the full row tiles of a
//                          range, with or without the fused halo exchange of the partitioned path
//   run_step<T>            picks between them (csrc/cheby.cu); every caller goes through it
#pragma once
#include <type_traits>
#include "common.cuh"
#include "gspb200.h"

namespace gsp {

constexpr int kMaxScales = 16;   // filters per launch whose coefficients are passed by value

// x_new = alpha (L x_cur) + beta x_cur + gamma x_old over a range of rows;
//   add_source == false: r_i (+)= ck[i] x_new             (reference order, approximations.py:107-109)
//   add_source == true : x_new += sum_i ck[i] r_i[row, :]  (Clenshaw form, r holds read-only sources)
// Blocks are (rows, nsig) row-major, r is (nscales, r_rows, nsig).  ck / c0 are host arrays read
// for i < nscales only, c0 and x_old only in the first step.  The matrix comes first, in CSR order,
// so that it can be brace-initialised: Step<T> s{nnz, indptr, indices, vals}.
template <typename T>
struct Step {
  // the matrix (nnz bounds the tiled kernel's CSR slab copies)
  int64_t nnz = 0;
  const int32_t* indptr = nullptr;
  const int32_t* indices = nullptr;
  const T* vals = nullptr;
  // the blocks
  const T* x_cur = nullptr;
  const T* x_old = nullptr;        // may alias x_new (row-local)
  T* x_new = nullptr;
  T* r = nullptr;
  int64_t r_rows = 0;
  int nsig = 0;
  // the coefficients
  bool first = false;              // r_i = c0[i]/2 x_cur + ck[i] x_new; no x_old
  double alpha = 0, beta = 0, gamma = 0;
  int nscales = 0;
  const double* ck = nullptr;
  const double* c0 = nullptr;
  bool add_source = false;
  bool reverse = false;            // tiled kernel: walk the tiles from the last to the first
  const int64_t* out_perm = nullptr;   // x_new row of local row i is out_perm[i] (NULL: i)
  const gsp_ring_plan* ring = nullptr; // neighbour rings of the matrix (tiled kernel, rows from 0)
};

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Whether the tiled kernel takes the full tiles of [rb, re): float32, a tile plan, tiles that
// start at a multiple of 4 rows, at most kMaxScales filters, and every block it copies by TMA or
// reads and writes as float4 aligned to 16 bytes.
template <typename T>
bool tiled_step_applies(const Step<T>& s, int64_t rb, const gsp_tile_plan* plan) {
  return std::is_same<T, float>::value && plan && plan->rows_per_tile > 0 && rb % 4 == 0 &&
         s.nscales <= kMaxScales && aligned16(s.indptr) && aligned16(s.indices) &&
         aligned16(s.vals) && aligned16(s.x_cur) && aligned16(s.x_new) && aligned16(s.r) &&
         (s.first || aligned16(s.x_old));
}

// One step over rows [rb, re).  Without a halo: the tiled kernel on the full tiles where
// tiled_step_applies, the row-group kernel on the rest.  With a halo (partitioned path, rb == 0):
// the boundary ("front") tiles with the halo-capable instantiation, then the interior tiles, then
// the row-group kernel on the < rows_per_tile remainder; GSP_ERR_UNSUPPORTED when the tiled kernel
// does not apply, since the row-group kernel neither waits, pushes nor publishes.
template <typename T>
int run_step(const Step<T>& s, int64_t rb, int64_t re, const gsp_tile_plan* plan,
             const gsp_halo_fusion* halo, cudaStream_t st);

// The row-group kernel on rows [rb, re): any nsig / nscales.
template <typename T>
int cheby_step(const Step<T>& s, int64_t rb, int64_t re, cudaStream_t st);

// The tiled kernel on the full tiles of [rb, re) (rb % 4 == 0); reports the rows done.  With a halo
// (rb == 0) it runs the halo-capable instantiation, whose first tiles wait, push and publish as
// gsp_halo_fusion says.
// With `pair`, one launch runs step s (A) and step *pair->second (B, the step that follows A) on
// the full tiles: see cheby_pair_tiled.  The two are middle Clenshaw steps of one source; B gathers
// the block A writes, which is neither of A's input blocks.
struct PairLaunch {
  const Step<float>* second;
  const int32_t* slots;      // 2 * tiles entries of gsp_cheby_pair_plan_host, in the walk direction
  const int32_t* nbr_ptr;
  const int32_t* nbr_idx;
  unsigned* tile_done;       // one counter per tile, zero before launch_index 1
  unsigned launch_index;     // 1, 2, ... over the launches that share tile_done
};
int cheby_step_tiled_f32(const Step<float>& s, int64_t rb, int64_t re, const gsp_tile_plan& plan,
                         const gsp_halo_fusion* halo, int64_t* rows_done, cudaStream_t st,
                         const PairLaunch* pair = nullptr);

// Forward recurrence (approximations.py:99-112), step k = 1 .. m-1 of coefficient rows c
// (nscales x m): T_k = (4/lmax) L T_{k-1} - 2 T_{k-1} - T_{k-2} and r_i += c_ik T_k; the first step
// forms T_1 = (2/lmax) L x - x and r_i = c_i0/2 x + c_i1 T_1.  ck / c0 receive nscales values.
template <typename T>
void forward_coefs(Step<T>& s, int k, int m, int nscales, double lmax, const double* c, double* ck,
                   double* c0) {
  for (int i = 0; i < nscales; ++i) {
    ck[i] = c[int64_t(i) * m + k];
    c0[i] = c[int64_t(i) * m];
  }
  s.first = k == 1;
  s.alpha = s.first ? 2.0 / lmax : 4.0 / lmax;
  s.beta = s.first ? -1.0 : -2.0;
  s.gamma = s.first ? 0.0 : -1.0;
  s.nscales = nscales;
  s.ck = ck;
  s.c0 = c0;
  s.add_source = false;
  // every other step walks the tiles backwards: the lines of T_{k-1} and r that the previous
  // step wrote last are still in L2 and are the first ones this step reads
  s.reverse = (k & 1) == 0;
}

// Clenshaw's recurrence for coefficient rows c (nsrc x m, K = m - 1) over source blocks s_i:
//   S_k = sum_i c_ik s_i,  b_k = S_k + 2 Lt b_{k+1} - b_{k+2},  out = S_0/2 + Lt b_1 - b_2,
// Lt = (2/lmax) L - I.  Sets the step that forms b_k (k = K-1 .. 0, b_0 = out) from
// x_cur = b_{k+1}, x_old = b_{k+2} and the sources in r.  With one source b_K = c_K x is never
// formed: b_{K-1} comes from x itself in the first form (with K == 1 that step is the output), and
// the next step folds -b_K into its source term.  Several sources start from b_K = S_K.
// ck receives nsrc values.
template <typename T>
void clenshaw_coefs(Step<T>& s, int k, int m, int nsrc, double lmax, const double* c, double* ck) {
  const int K = m - 1;
  const double a2 = 4.0 / lmax;                  // 2 Lt = a2 L - 2 I
  const bool last = k == 0;
  s.c0 = nullptr;
  if (nsrc == 1 && k == K - 1) {
    s.first = true;
    s.nscales = 0;
    s.ck = nullptr;
    s.add_source = false;
    s.reverse = false;
    s.gamma = 0.0;
    if (K == 1) {                                // out = c0/2 x + c1 Lt x
      s.alpha = c[1] * 2.0 / lmax;
      s.beta = 0.5 * c[0] - c[1];
    } else {                                     // b_{K-1} = c_{K-1} x + 2 Lt (c_K x)
      s.alpha = c[K] * a2;
      s.beta = c[K - 1] - 2.0 * c[K];
    }
    return;
  }
  // middle: b_k = a2 L b_{k+1} - 2 b_{k+1} - b_{k+2} + S_k
  // last  : out = (a2/2) L b_1 - b_1 - b_2 + S_0/2
  s.first = false;
  s.alpha = last ? 0.5 * a2 : a2;
  s.beta = last ? -1.0 : -2.0;
  s.gamma = -1.0;
  for (int i = 0; i < nsrc; ++i) ck[i] = (last ? 0.5 : 1.0) * c[int64_t(i) * m + k];
  if (k + 2 > (nsrc == 1 ? K - 1 : K)) {
    // no b_{k+2} block: it is c_K x (one source, folded into the source term) or 0
    if (nsrc == 1) ck[0] -= c[K];
    s.gamma = 0.0;
  }
  s.nscales = nsrc;
  s.ck = ck;
  s.add_source = true;
  s.reverse = (k & 1) == 0;
}

}  // namespace gsp
