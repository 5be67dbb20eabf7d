// Fixed-order reductions shared by the accelerated proximal solvers (csrc/simplex.cu, csrc/tv.cu).
#pragma once
#include "common.cuh"

namespace gsp {

// grid of a pass that strides over n items, rpb per block: four blocks per SM at most, and at most
// max_blocks (the size of the caller's per-block partials area)
static inline int pass_blocks(int64_t n, int rpb, int max_blocks) {
  return (int)std::max<int64_t>(
      1, std::min<int64_t>(ceil_div(n, rpb), std::min<int64_t>(int64_t(sm_count()) * 4, max_blocks)));
}

// sum over the w lanes of an aligned power-of-two sub-warp (xor butterfly: fixed order)
template <typename S>
__device__ __forceinline__ S group_sum(S v, int w) {
  for (int off = w >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

}  // namespace gsp
