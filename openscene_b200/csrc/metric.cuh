// Intersection / union / target counting of util/util.py:132-145 for one (output, target) pair, shared by
// k_inter_union (csrc/metric.cu) and the cross-entropy epilogue of the tensor-core match (csrc/match_tc.cu).
#pragma once
#include <cuda_runtime.h>

namespace osb {

// bins: [3, K] = intersection | output | target, in shared (uint32) or global (unsigned long long) memory
template <typename B>
__device__ __forceinline__ void inter_union_add(long long o, long long t, int K, int ignore_id, B *bins) {
  if (t == ignore_id) o = ignore_id;                   // util.py:138 output[target == ignore_index] = ignore_index
  const bool o_in = o >= 0 && o < K, t_in = t >= 0 && t < K;     // histc(bins=K, min=0, max=K-1) drops the rest
  if (o_in && o == t) atomicAdd(&bins[o], B(1));
  if (o_in) atomicAdd(&bins[K + o], B(1));
  if (t_in) atomicAdd(&bins[2 * K + t], B(1));
}

}  // namespace osb
