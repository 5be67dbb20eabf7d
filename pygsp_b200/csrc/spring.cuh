// Pieces of the Fruchterman-Reingold step shared by the all-pairs repulsion (csrc/layout.cu) and
// the Barnes-Hut repulsion (csrc/barnes_hut.cu): the clamped reciprocal 1 / max(d^2, 0.01^2) and
// the update kernel that adds the repulsion partials, the attraction over W's CSR and moves the
// vertices (DESIGN.md 4.14, 4.24).
#pragma once
#include <math.h>

#include "common.cuh"

namespace gsp {
namespace spring {

constexpr double kMinD2 = 0.01 * 0.01;

// 1 / max(d2, 0.01^2); a compare and select rather than fmax, whose NaN handling costs four
// integer instructions per pair (a NaN d2 gives a NaN result either way)
__device__ __forceinline__ double inv_d2(double d2) {
  const double x = d2 < kMinD2 ? kMinD2 : d2;
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  const double e = fma(-x, r, 1.0);
  return fma(r, fma(e, e, e), r);
}

// disp_i = (partials in chunk order) - sum_{j in row i, w_ij > 0} delta_ij d_ij / k, accumulated
// in partial[0][i][:]; then pos_out[i] = pos_in[i] + disp_i t / length_i (fixed: disp_i = 0)
template <typename T>
__global__ void spring_update_kernel(int64_t n, int dim, const int32_t* __restrict__ indptr,
                                     const int32_t* __restrict__ indices,
                                     const T* __restrict__ data, double k, double t,
                                     const uint8_t* __restrict__ fixed, int64_t n_chunks,
                                     const double* __restrict__ pos_in, double* partial,
                                     double* __restrict__ pos_out) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double* p = pos_in + i * dim;
  double* disp = partial + i * dim;
  if (fixed != nullptr && fixed[i]) {
    for (int a = 0; a < dim; ++a) pos_out[i * dim + a] = p[a];
    return;
  }
  for (int64_t c = 1; c < n_chunks; ++c)
    for (int a = 0; a < dim; ++a) disp[a] += partial[(c * n + i) * dim + a];
  for (int e = indptr[i]; e < indptr[i + 1]; ++e) {
    if (!(data[e] > T(0))) continue;
    const double* q = pos_in + int64_t(indices[e]) * dim;
    double d2 = 0.0;
    for (int a = 0; a < dim; ++a) {
      const double dl = p[a] - q[a];
      d2 = a == 0 ? dl * dl : fma(dl, dl, d2);
    }
    const double g = fmax(sqrt(d2), 0.01) / k;
    for (int a = 0; a < dim; ++a) disp[a] = fma(-(p[a] - q[a]), g, disp[a]);
  }
  double len2 = 0.0;
  for (int a = 0; a < dim; ++a) len2 = a == 0 ? disp[a] * disp[a] : fma(disp[a], disp[a], len2);
  double length = sqrt(len2);
  if (length < 0.01) length = 0.1;
  for (int a = 0; a < dim; ++a) pos_out[i * dim + a] = p[a] + disp[a] * t / length;
}

}  // namespace spring
}  // namespace gsp
