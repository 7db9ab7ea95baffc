// Running argmax of the test-time repeat vote (csrc/vote.cu, the vote epilogue of csrc/match_tc.cu) and of the validation
// cross-entropy epilogue (k_match_tc_ce).
//
// The evaluation drivers take labels with torch's CPU `x.float().max(1)[1]` (run/evaluate.py:400, run/eval_mink.py:205):
// a row holding a NaN takes the index of its first NaN; otherwise the first maximum wins (-0 == +0, ties go to the lowest
// index, inf beats every finite value).  The existing match label (first maximum among non-NaN values) is a different
// rule and stays as it is.
#pragma once
#include <cuda_runtime.h>

namespace osb {

struct VoteArgmax {
  float v;
  int k;   // < 0: no column seen yet

  __device__ __forceinline__ void init() { v = 0.f; k = -1; }

  // columns arrive in ascending order within one thread
  __device__ __forceinline__ void take(float x, int kx) {
    if (k < 0 || (v == v && (x != x || x > v))) { v = x; k = kx; }
  }

  // merge the state of another thread (columns in any order)
  __device__ __forceinline__ void merge(float ov, int ok) {
    if (ok < 0) return;
    if (k < 0) { v = ov; k = ok; return; }
    const bool n = v != v, on = ov != ov;
    bool win;
    if (n || on) win = on && (!n || ok < k);
    else win = ov > v || (ov == v && ok < k);
    if (win) { v = ov; k = ok; }
  }

  // reduce over each group of WIDTH consecutive lanes (all lanes of the warp take part)
  template <int WIDTH>
  __device__ __forceinline__ void reduce() {
#pragma unroll
    for (int o = 1; o < WIDTH; o <<= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, v, o);
      const int ok = __shfl_xor_sync(0xffffffffu, k, o);
      merge(ov, ok);
    }
  }
};

}  // namespace osb
