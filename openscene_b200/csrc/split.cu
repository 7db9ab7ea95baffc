// fp32 <-> split-bf16 rows (the activation layout of the tensor-core path, see include/osb200.h).
#include "common.cuh"
#include <algorithm>

namespace osb {

// one thread converts 8 consecutive channels: reads 32 B fp32, writes 16 B hi + 16 B lo
__global__ void k_f32_to_split(const float *__restrict__ in, int64_t n, int c, uint8_t *__restrict__ out) {
  const int64_t groups = n * (c / 8);
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = g / (c / 8);
    const int c0 = (int)(g - r * (c / 8)) * 8;
    const float4 a = __ldg(reinterpret_cast<const float4 *>(in + r * c + c0));
    const float4 b = __ldg(reinterpret_cast<const float4 *>(in + r * c + c0 + 4));
    const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    __align__(16) __nv_bfloat16 hi[8], lo[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) split_bf16(v[j], hi[j], lo[j]);
    uint8_t *row = out + r * (int64_t)c * 4 + split_off_hi(c0);
    *reinterpret_cast<uint4 *>(row) = *reinterpret_cast<const uint4 *>(hi);
    *reinterpret_cast<uint4 *>(row + 64) = *reinterpret_cast<const uint4 *>(lo);
  }
}

__global__ void k_split_to_f32(const uint8_t *__restrict__ in, int64_t n, int c, float *__restrict__ out) {
  const int64_t groups = n * (c / 8);
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = g / (c / 8);
    const int c0 = (int)(g - r * (c / 8)) * 8;
    const uint8_t *row = in + r * (int64_t)c * 4 + split_off_hi(c0);
    __align__(16) __nv_bfloat16 hi[8], lo[8];
    *reinterpret_cast<uint4 *>(hi) = __ldg(reinterpret_cast<const uint4 *>(row));
    *reinterpret_cast<uint4 *>(lo) = __ldg(reinterpret_cast<const uint4 *>(row + 64));
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = join_bf16(hi[j], lo[j]);
    *reinterpret_cast<float4 *>(out + r * c + c0) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4 *>(out + r * c + c0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
}

}  // namespace osb

using namespace osb;

extern "C" {

int osb_f32_to_split(const float *in, int64_t n, int32_t c, void *out_split, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(c > 0 && c % 32 == 0, "osb_f32_to_split: channels (%d) must be a multiple of 32", c);
  if (n == 0) return 0;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n * (c / 8), 256), 132 * 16);
  k_f32_to_split<<<grid, 256, 0, stream>>>(in, n, c, (uint8_t *)out_split);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_split_to_f32(const void *in_split, int64_t n, int32_t c, float *out, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(c > 0 && c % 32 == 0, "osb_split_to_f32: channels (%d) must be a multiple of 32", c);
  if (n == 0) return 0;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n * (c / 8), 256), 132 * 16);
  k_split_to_f32<<<grid, 256, 0, stream>>>((const uint8_t *)in_split, n, c, out);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// SM clock measured on the device: cycles of clock64() per nanosecond of %globaltimer over ~20 us.
// bench.py calls it between timed steps: an NVML / nvidia-smi query during the timed region stalls the GPU for
// tens of milliseconds, this costs one 20 us single-thread kernel outside every step's event pair.
namespace osb {
__global__ void k_measure_sm_mhz(float *__restrict__ out) {
  unsigned long long t0, t1;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  const long long c0 = clock64();
  do { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); } while (t1 - t0 < 20000ull);
  const long long c1 = clock64();
  *out = (float)((double)(c1 - c0) * 1000.0 / (double)(t1 - t0));
}
}  // namespace osb

extern "C" int osb_measure_sm_mhz(float *mhz_dev, void *stream_) {
  OSB_CHECK(mhz_dev != nullptr, "osb_measure_sm_mhz: null output");
  osb::k_measure_sm_mhz<<<1, 1, 0, (cudaStream_t)stream_>>>(mhz_dev);
  OSB_LAUNCH_CHECK();
  return 0;
}
