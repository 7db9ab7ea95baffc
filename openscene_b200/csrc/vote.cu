// Test-time repeat vote on CUDA cores (run/evaluate.py:385-425, run/eval_mink.py:167-216).
//
//   store[p, k] = store[p, k] + src[v(p), k]        v(p) = inds_reverse[p], or p when NULL
//   label_cur[p] = argmax_k src[v(p), k],  label_acc[p] = argmax_k store[p, k]      (vote.cuh: torch CPU max(1)[1])
//
// in the store's own precision: one fp16 add rounded to nearest even (the reference's `store = pred + store` on fp16 CPU
// tensors), or one fp32 add (eval_mink's fp32 logits).  This is the eval_mink path, the OSB_MATCH_SIMT=1 route of the
// match vote, and the independent cross-check of the vote epilogue in csrc/match_tc.cu.  One warp per point: K * (2 or
// 4) bytes read from src and read + written in the store per point, nothing else.
#include "common.cuh"
#include "vote.cuh"

#include <algorithm>

namespace osb {

__device__ __forceinline__ __half vote_add(__half a, __half b) { return __hadd(a, b); }
__device__ __forceinline__ float vote_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float vote_f32(__half a) { return __half2float(a); }
__device__ __forceinline__ float vote_f32(float a) { return a; }

template <typename T>
__global__ void __launch_bounds__(256)
k_vote_accumulate(const T *__restrict__ src, const int64_t *__restrict__ inds_reverse, int64_t n_pts, int k_cls,
                  T *__restrict__ store, int64_t *__restrict__ label_cur, int64_t *__restrict__ label_acc) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t p = warp; p < n_pts; p += nwarps) {
    const int64_t v = inds_reverse ? __ldg(inds_reverse + p) : p;
    const T *s = src + v * k_cls;
    T *st = store + p * k_cls;
    VoteArgmax cur, acc;
    cur.init();
    acc.init();
    for (int k = lane; k < k_cls; k += 32) {
      const T x = s[k];
      const T sum = vote_add(st[k], x);
      st[k] = sum;
      cur.take(vote_f32(x), k);
      acc.take(vote_f32(sum), k);
    }
    cur.reduce<32>();
    acc.reduce<32>();
    if (lane == 0) {
      if (label_cur) label_cur[p] = cur.k;
      if (label_acc) label_acc[p] = acc.k;
    }
  }
}

int vote_accumulate_run(const void *src, int src_is_f16, const int64_t *inds_reverse, int64_t n_pts, int k, void *store,
                        int64_t *label_cur, int64_t *label_acc, cudaStream_t stream) {
  if (n_pts == 0) return 0;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n_pts, 8), 132 * 8);
  if (src_is_f16)
    k_vote_accumulate<__half><<<grid, 256, 0, stream>>>((const __half *)src, inds_reverse, n_pts, k, (__half *)store,
                                                        label_cur, label_acc);
  else
    k_vote_accumulate<float><<<grid, 256, 0, stream>>>((const float *)src, inds_reverse, n_pts, k, (float *)store,
                                                       label_cur, label_acc);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // namespace osb

extern "C" int osb_vote_accumulate(const void *src, int32_t src_is_f16, int64_t n_src, const int64_t *inds_reverse,
                                   int64_t n_pts, int32_t k, void *store, int64_t *label_cur, int64_t *label_acc,
                                   void *stream_) {
  OSB_CHECK(k >= 1 && k <= 512, "osb_vote_accumulate: K=%d outside 1..512", k);
  OSB_CHECK(n_src > 0 && n_pts >= 0, "osb_vote_accumulate: bad shape (n_src=%lld, n_pts=%lld)", (long long)n_src,
            (long long)n_pts);
  OSB_CHECK(inds_reverse != nullptr || n_src == n_pts,
            "osb_vote_accumulate: without inds_reverse the source needs one row per point (n_src=%lld, n_pts=%lld)",
            (long long)n_src, (long long)n_pts);
  OSB_CHECK(src != nullptr && store != nullptr, "osb_vote_accumulate: null source or store");
  return osb::vote_accumulate_run(src, src_is_f16, inds_reverse, n_pts, k, store, label_cur, label_acc,
                                  (cudaStream_t)stream_);
}
