// Device helpers shared by the fp32 CUDA-core distillation heads (cos_head.cu, l1_head.cu): split-row staging and the
// 4 x 4 register tile of their products.
#pragma once
#include "common.cuh"

namespace osb {

// channels 8 q .. 8 q + 7 of a 128-byte split line
__device__ inline void head_load8(const uint8_t *line, int q, float v[8]) {
  union { uint4 u; __nv_bfloat16 b[8]; } hi, lo;
  hi.u = __ldg(reinterpret_cast<const uint4 *>(line + 16 * q));
  lo.u = __ldg(reinterpret_cast<const uint4 *>(line + 64 + 16 * q));
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = join_bf16(hi.b[j], lo.b[j]);
}

// acc[e][f] += a[e] b[f]
__device__ inline void head_fma44(float acc[4][4], const float4 a, const float4 b) {
  const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int f = 0; f < 4; ++f) acc[e][f] = fmaf(av[e], bv[f], acc[e][f]);
}

}  // namespace osb
