// Segmentation metrics accumulated on the device (SURVEY.md 8f rank 4): the confusion matrix of util/metric.py:9-25
// and the intersection / union / target histograms of util/util.py:132-145 (which round-trips through .cpu() for
// torch.histc).  Integer counting: per-block shared-memory histograms, flushed with 64-bit atomics.
#include "common.cuh"
#include "metric.cuh"

#include <algorithm>

namespace osb {

template <typename T>
__global__ void __launch_bounds__(256)
k_confusion(const T *__restrict__ pred, const T *__restrict__ gt, int64_t n, int C, int ignore_id, int nofeat_id,
            unsigned long long *__restrict__ conf, int use_smem, int32_t *__restrict__ bad) {
  extern __shared__ uint32_t s_bins[];
  const int W = C + 1, bins = W * W;
  if (use_smem) {
    for (int b = threadIdx.x; b < bins; b += blockDim.x) s_bins[b] = 0;
    __syncthreads();
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const long long g = (long long)gt[i];
    if (g == ignore_id) continue;                       // metric.py:13 idxs = gt_ids != UNKNOWN_ID
    long long p = (long long)pred[i];
    if (p == nofeat_id) p = C;                          // metric.py:15 "no feature" -> extra row
    if (p < 0 || p > C || g < 0 || g >= C) { atomicAdd(bad, 1); continue; }
    const int b = (int)p * W + (int)g;                  // rows = prediction, columns = ground truth
    if (use_smem) atomicAdd(&s_bins[b], 1u);
    else atomicAdd(&conf[b], 1ull);
  }
  if (use_smem) {
    __syncthreads();
    for (int b = threadIdx.x; b < bins; b += blockDim.x)
      if (s_bins[b]) atomicAdd(&conf[b], (unsigned long long)s_bins[b]);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
k_inter_union(const T *__restrict__ out, const T *__restrict__ tgt, int64_t n, int K, int ignore_id,
              unsigned long long *__restrict__ areas, int use_smem) {
  extern __shared__ uint32_t s_bins[];
  if (use_smem) {
    for (int b = threadIdx.x; b < 3 * K; b += blockDim.x) s_bins[b] = 0;
    __syncthreads();
  }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const long long t = (long long)tgt[i], o = (long long)out[i];
    if (use_smem) inter_union_add(o, t, K, ignore_id, s_bins);
    else inter_union_add(o, t, K, ignore_id, areas);
  }
  if (use_smem) {
    __syncthreads();
    for (int b = threadIdx.x; b < 3 * K; b += blockDim.x)
      if (s_bins[b]) atomicAdd(&areas[b], (unsigned long long)s_bins[b]);
  }
}

constexpr size_t kMetricSmemMax = 200 * 1024;

}  // namespace osb

using namespace osb;

extern "C" {

int osb_confusion_accumulate(const void *pred, const void *gt, int32_t labels_are_i64, int64_t n, int32_t num_classes,
                             int32_t ignore_id, int32_t nofeat_id, uint64_t *confusion, int32_t *bad_labels, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(num_classes > 0 && num_classes < 4096, "osb_confusion_accumulate: num_classes %d out of range", num_classes);
  OSB_CHECK(confusion && bad_labels, "osb_confusion_accumulate: null output");
  if (n == 0) return 0;
  const size_t smem = (size_t)(num_classes + 1) * (num_classes + 1) * sizeof(uint32_t);
  const int use_smem = smem <= kMetricSmemMax;
  // a block's uint32 bins must not overflow: every block sees at most ceil(n / grid) * ... < 2^32 items for n < 2^40
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n, 256 * 8), 132 * 4);
  auto *conf = reinterpret_cast<unsigned long long *>(confusion);
  if (labels_are_i64) {
    if (use_smem) OSB_CUDA(cudaFuncSetAttribute(k_confusion<int64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMetricSmemMax));
    k_confusion<int64_t><<<grid, 256, use_smem ? smem : 0, stream>>>((const int64_t *)pred, (const int64_t *)gt, n, num_classes, ignore_id,
                                                                     nofeat_id, conf, use_smem, bad_labels);
  } else {
    if (use_smem) OSB_CUDA(cudaFuncSetAttribute(k_confusion<int32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMetricSmemMax));
    k_confusion<int32_t><<<grid, 256, use_smem ? smem : 0, stream>>>((const int32_t *)pred, (const int32_t *)gt, n, num_classes, ignore_id,
                                                                     nofeat_id, conf, use_smem, bad_labels);
  }
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_intersection_union(const void *output, const void *target, int32_t labels_are_i64, int64_t n, int32_t K,
                           int32_t ignore_id, uint64_t *areas, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(K > 0 && K < (1 << 20), "osb_intersection_union: K %d out of range", K);
  OSB_CHECK(areas, "osb_intersection_union: null output");
  if (n == 0) return 0;
  const size_t smem = (size_t)3 * K * sizeof(uint32_t);
  const int use_smem = smem <= 48 * 1024;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n, 256 * 8), 132 * 4);
  auto *a = reinterpret_cast<unsigned long long *>(areas);
  if (labels_are_i64)
    k_inter_union<int64_t><<<grid, 256, use_smem ? smem : 0, stream>>>((const int64_t *)output, (const int64_t *)target, n, K, ignore_id, a, use_smem);
  else
    k_inter_union<int32_t><<<grid, 256, use_smem ? smem : 0, stream>>>((const int32_t *)output, (const int32_t *)target, n, K, ignore_id, a, use_smem);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
