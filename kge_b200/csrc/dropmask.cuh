// dropmask.cuh — the keep multipliers of one dropout draw (layout: include/b200kge.h), regenerated where an operand is
// loaded: shared by the negative-sampling dropout kernels (ns_dropout.cu) and the masked instantiations of ns_kernel
// (rowwise.cu) and ns_backward_kernel (grad.cu).
#pragma once
#include "common.cuh"
#include "philox.cuh"

namespace b200kge {

// multipliers (1 / (1 - p) or 0) of elements k..k+3 of mask row `mrow` (k % 4 == 0, width % 4 == 0: one Philox block)
__device__ __forceinline__ void drop_mask4(const DropMask& m, uint64_t mrow, int width, int k, float (&mk)[4]) {
  if (m.thresh >= (1ull << 32)) { mk[0] = mk[1] = mk[2] = mk[3] = 1.f; return; }
  const uint64_t g = (mrow * (uint64_t)width + (uint64_t)k) >> 2;
  const uint64_t c = ((uint64_t)m.stream << 46) | g;
  uint32_t w[4] = {(uint32_t)c, (uint32_t)(c >> 32), (uint32_t)m.call, (uint32_t)(m.call >> 32)};
  philox4x32_10(w, m.seed);
#pragma unroll
  for (int j = 0; j < 4; ++j) mk[j] = ((uint64_t)w[j] < m.thresh) ? m.scale : 0.f;
}

// multiplier of one element
__device__ __forceinline__ float drop_mask1(const DropMask& m, uint64_t mrow, int width, int k) {
  if (m.thresh >= (1ull << 32)) return 1.f;
  const uint64_t e = mrow * (uint64_t)width + (uint64_t)k;
  const uint64_t c = ((uint64_t)m.stream << 46) | (e >> 2);
  uint32_t w[4] = {(uint32_t)c, (uint32_t)(c >> 32), (uint32_t)m.call, (uint32_t)(m.call >> 32)};
  philox4x32_10(w, m.seed);
  return ((uint64_t)w[e & 3] < m.thresh) ? m.scale : 0.f;
}

}  // namespace b200kge
