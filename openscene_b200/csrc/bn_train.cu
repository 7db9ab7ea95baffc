// Train-mode BatchNorm on split rows (nn.BatchNorm1d.forward with training=True over the [n, C] feature matrix):
//   osb_bn_batch_stats   per-channel mean / biased variance over all n rows, scale = w / sqrt(var + eps),
//                        shift = b - mean * scale, and the running-buffer update of torch.nn.modules.batchnorm;
//   osb_bn_apply_split   y = act(x * scale + shift + r) in place, r = none | res | res * res_scale + res_shift.
//   osb_bn_batch_stats_save / osb_bn_apply_split_out: the same, also keeping the batch mean / invstd and the raw rows (training);
//   osb_bn_backward_reduce / osb_bn_backward_apply: the backward of act(BN(z) + r) (autograd of F.batch_norm(training=True)).
//
// Statistics: every value is shifted by the channel's value in row 0 and the shifted sums and sums of squares are accumulated in
// fp64, so the variance does not cancel against a mean that is large compared with the spread (activations after ReLU and
// residual adds).  Blocks write per-channel partials to the workspace and one block merges them in a fixed order: the result
// is bit-reproducible and no float atomics are used.
//
// Thread mapping (both passes): 8 threads cover one 128-byte line [hi x32 | lo x32] of a row, each 4 channels (8 bytes of hi
// and the matching 8 bytes of lo), so every warp load / store covers whole lines of four rows.
#include "common.cuh"
#include <algorithm>
#include <math.h>

namespace osb {

constexpr int BN_THREADS = 256;            // 32 row slots x 8 threads per line
constexpr int BN_ROW_SLOTS = BN_THREADS / 8;
constexpr int64_t BN_ROWS_PER_BLOCK = 512;
constexpr int64_t BN_MAX_ROW_BLOCKS = 1024;

// row blocks of the partial pass: a function of n only, so the workspace size and the merge order never depend on the device
static int64_t bn_row_blocks(int64_t n) { return std::min<int64_t>(ceil_div(n, BN_ROWS_PER_BLOCK), BN_MAX_ROW_BLOCKS); }

__device__ inline void load4(const uint8_t *line, int q, float v[4]) {
  union { uint2 u; __nv_bfloat16 b[4]; } h, l;
  h.u = *reinterpret_cast<const uint2 *>(line + 8 * q);
  l.u = *reinterpret_cast<const uint2 *>(line + 64 + 8 * q);
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = join_bf16(h.b[j], l.b[j]);
}

__device__ inline void store4(uint8_t *line, int q, const float v[4]) {
  union { uint2 u; __nv_bfloat16 b[4]; } h, l;
#pragma unroll
  for (int j = 0; j < 4; ++j) split_bf16(v[j], h.b[j], l.b[j]);
  *reinterpret_cast<uint2 *>(line + 8 * q) = h.u;
  *reinterpret_cast<uint2 *>(line + 64 + 8 * q) = l.u;
}

// grid (row blocks, C/32).  part: [row block][2][C] fp64 = (sum of x - x[0], sum of (x - x[0])^2)
__global__ void __launch_bounds__(BN_THREADS) k_bn_partial(const uint8_t *__restrict__ x, int64_t n, int c, double *__restrict__ part) {
  __shared__ double s1[BN_ROW_SLOTS][32], s2[BN_ROW_SLOTS][32];
  const int q = threadIdx.x & 7, slot = threadIdx.x >> 3, g = blockIdx.y;
  const int64_t row_bytes = (int64_t)c * 4;
  const int64_t rpb = (n + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = (int64_t)blockIdx.x * rpb, r1 = min(n, r0 + rpb);
  const uint8_t *base = x + (int64_t)g * 128;
  float pivot[4];
  load4(base, q, pivot);
  double a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0};
#pragma unroll 4
  for (int64_t r = r0 + slot; r < r1; r += BN_ROW_SLOTS) {
    float v[4];
    load4(base + r * row_bytes, q, v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double d = (double)v[j] - (double)pivot[j];
      a1[j] += d;
      a2[j] = fma(d, d, a2[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { s1[slot][4 * q + j] = a1[j]; s2[slot][4 * q + j] = a2[j]; }
  __syncthreads();
  if (threadIdx.x < 64) {                                   // fixed-order merge of the 32 row slots
    const int ch = threadIdx.x & 31;
    double (*s)[32] = threadIdx.x < 32 ? s1 : s2;
    double acc = 0;
    for (int i = 0; i < BN_ROW_SLOTS; ++i) acc += s[i][ch];
    part[((int64_t)blockIdx.x * 2 + (threadIdx.x >> 5)) * c + g * 32 + ch] = acc;
  }
}

// one block: merge the partials of every channel in a fixed order, write scale / shift, move the running buffers
__global__ void __launch_bounds__(BN_THREADS) k_bn_finalize(const uint8_t *__restrict__ x, int64_t n, int c, int64_t nblk,
                                                            const double *__restrict__ part, const float *__restrict__ weight,
                                                            const float *__restrict__ bias, double eps, double momentum,
                                                            float *running_mean, float *running_var, int64_t *num_batches_tracked,
                                                            float *__restrict__ scale, float *__restrict__ shift,
                                                            float *__restrict__ mean_out, float *__restrict__ invstd_out) {
  __shared__ double m1[8][32], m2[8][32];
  const int ch = threadIdx.x & 31, slot = threadIdx.x >> 5;
  const int64_t tracked = *num_batches_tracked + 1;          // read by every thread before thread 0 writes it (barriers below)
  // nn.BatchNorm1d: momentum None -> cumulative average with factor 1 / num_batches_tracked, read after the increment
  const double m = momentum < 0 ? 1.0 / (double)tracked : momentum;
  for (int g = 0; g < c / 32; ++g) {
    const int cc = g * 32 + ch;
    double a1 = 0, a2 = 0;
    for (int64_t b = slot; b < nblk; b += 8) {
      a1 += part[(b * 2) * c + cc];
      a2 += part[(b * 2 + 1) * c + cc];
    }
    m1[slot][ch] = a1;
    m2[slot][ch] = a2;
    __syncthreads();
    if (threadIdx.x < 32) {
      double t1 = 0, t2 = 0;
      for (int i = 0; i < 8; ++i) { t1 += m1[i][ch]; t2 += m2[i][ch]; }
      const uint8_t *row0 = x + split_off_hi(cc);
      const double pivot = (double)join_bf16(*reinterpret_cast<const __nv_bfloat16 *>(row0),
                                             *reinterpret_cast<const __nv_bfloat16 *>(row0 + 64));
      const double dm = t1 / (double)n;
      const double v = t2 / (double)n - dm * dm;
      const double var = v < 0.0 ? 0.0 : v;                          // biased: what normalises the batch; NaN stays NaN
      const double mean = pivot + dm;
      const double istd = 1.0 / sqrt(var + eps);
      const double sc = (double)weight[cc] * istd;
      if (mean_out) { mean_out[cc] = (float)mean; invstd_out[cc] = (float)istd; }
      scale[cc] = (float)sc;
      shift[cc] = (float)((double)bias[cc] - mean * sc);
      running_mean[cc] = (float)((1.0 - m) * (double)running_mean[cc] + m * mean);
      running_var[cc] = (float)((1.0 - m) * (double)running_var[cc] + m * var * (double)n / (double)(n - 1));   // unbiased
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *num_batches_tracked = tracked;
}

// torch.relu: NaN passes through (fmaxf would turn it into 0); otherwise the same instruction as fmaxf(y, 0)
__device__ inline float relu_nan(float y) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(y), "f"(0.f));
  return r;
}

// grid (row chunks, C/32): RES 0 = no residual, 1 = split rows, 2 = split rows normalised by res_scale / res_shift
template <int RES, bool RELU>
__global__ void __launch_bounds__(BN_THREADS) k_bn_apply(const uint8_t *x, uint8_t *y_out, int64_t n, int c, const float *__restrict__ scale,
                                                         const float *__restrict__ shift, const uint8_t *__restrict__ res,
                                                         const float *__restrict__ res_scale, const float *__restrict__ res_shift) {
  const int q = threadIdx.x & 7, g = blockIdx.y;
  const int ch = g * 32 + 4 * q;
  const int64_t row_bytes = (int64_t)c * 4;
  float sc[4], sh[4], rsc[4], rsh[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    sc[j] = __ldg(scale + ch + j);
    sh[j] = __ldg(shift + ch + j);
    if (RES == 2) { rsc[j] = __ldg(res_scale + ch + j); rsh[j] = __ldg(res_shift + ch + j); }
  }
  for (int64_t r = (int64_t)blockIdx.x * BN_ROW_SLOTS + (threadIdx.x >> 3); r < n; r += (int64_t)gridDim.x * BN_ROW_SLOTS) {
    const int64_t off = r * row_bytes + (int64_t)g * 128;
    float v[4], rv[4];
    load4(x + off, q, v);
    if (RES) load4(res + r * row_bytes + (int64_t)g * 128, q, rv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float y = fmaf(v[j], sc[j], sh[j]);
      if (RES == 1) y += rv[j];
      if (RES == 2) y += fmaf(rv[j], rsc[j], rsh[j]);
      v[j] = RELU ? relu_nan(y) : y;
    }
    store4(y_out + off, q, v);
  }
}

template <int RES, bool RELU>
static void launch_apply(dim3 grid, cudaStream_t st, const void *x, void *y, int64_t n, int c, const float *scale,
                         const float *shift, const void *res, const float *res_scale, const float *res_shift) {
  k_bn_apply<RES, RELU><<<grid, BN_THREADS, 0, st>>>((const uint8_t *)x, (uint8_t *)y, n, c, scale, shift, (const uint8_t *)res,
                                                     res_scale, res_shift);
}

// ---- backward of y = act(BN(z) + r), BN with batch statistics: g' = g [not y <= 0] (torch's threshold_backward: a NaN output
//      passes its gradient; g without ReLU), x^ = (z - mean) invstd,
//      dbias = sum g', dweight = sum g' x^, dz = weight invstd (g' - sum g' / n - x^ sum g' x^ / n)

// grid (row blocks, C/32).  part: [row block][2][C] fp64 = (sum of g', sum of g' x^)
template <bool MASK>
__global__ void __launch_bounds__(BN_THREADS) k_bn_bwd_partial(const uint8_t *__restrict__ y, const uint8_t *__restrict__ gr,
                                                               const uint8_t *__restrict__ z, int64_t n, int c,
                                                               const float *__restrict__ mean, const float *__restrict__ invstd,
                                                               double *__restrict__ part) {
  __shared__ double s1[BN_ROW_SLOTS][32], s2[BN_ROW_SLOTS][32];
  const int q = threadIdx.x & 7, slot = threadIdx.x >> 3, g = blockIdx.y;
  const int64_t row_bytes = (int64_t)c * 4;
  const int64_t rpb = (n + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = (int64_t)blockIdx.x * rpb, r1 = min(n, r0 + rpb);
  double mu[4], is[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) { mu[j] = __ldg(mean + g * 32 + 4 * q + j); is[j] = __ldg(invstd + g * 32 + 4 * q + j); }
  double a1[4] = {0, 0, 0, 0}, a2[4] = {0, 0, 0, 0};
#pragma unroll 2
  for (int64_t r = r0 + slot; r < r1; r += BN_ROW_SLOTS) {
    const int64_t off = r * row_bytes + (int64_t)g * 128;
    float gv[4], zv[4], yv[4];
    load4(gr + off, q, gv);
    load4(z + off, q, zv);
    if (MASK) load4(y + off, q, yv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const double gp = (MASK && yv[j] <= 0.f) ? 0.0 : (double)gv[j];
      a1[j] += gp;
      a2[j] = fma(gp, ((double)zv[j] - mu[j]) * is[j], a2[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { s1[slot][4 * q + j] = a1[j]; s2[slot][4 * q + j] = a2[j]; }
  __syncthreads();
  if (threadIdx.x < 64) {                                   // fixed-order merge of the 32 row slots
    const int ch = threadIdx.x & 31;
    double (*s)[32] = threadIdx.x < 32 ? s1 : s2;
    double acc = 0;
    for (int i = 0; i < BN_ROW_SLOTS; ++i) acc += s[i][ch];
    part[((int64_t)blockIdx.x * 2 + (threadIdx.x >> 5)) * c + g * 32 + ch] = acc;
  }
}

// one block: merge the partials in a fixed order -> sums [2][c] and the affine gradients (written or accumulated)
__global__ void __launch_bounds__(BN_THREADS) k_bn_bwd_finalize(int c, int64_t nblk, const double *__restrict__ part,
                                                                float *__restrict__ sums, float *dweight, float *dbias,
                                                                int accumulate) {
  __shared__ double m1[8][32], m2[8][32];
  const int ch = threadIdx.x & 31, slot = threadIdx.x >> 5;
  for (int g = 0; g < c / 32; ++g) {
    const int cc = g * 32 + ch;
    double a1 = 0, a2 = 0;
    for (int64_t b = slot; b < nblk; b += 8) {
      a1 += part[(b * 2) * c + cc];
      a2 += part[(b * 2 + 1) * c + cc];
    }
    m1[slot][ch] = a1;
    m2[slot][ch] = a2;
    __syncthreads();
    if (threadIdx.x < 32) {
      double t1 = 0, t2 = 0;
      for (int i = 0; i < 8; ++i) { t1 += m1[i][ch]; t2 += m2[i][ch]; }
      sums[cc] = (float)t1;
      sums[c + cc] = (float)t2;
      dbias[cc] = accumulate ? (float)((double)dbias[cc] + t1) : (float)t1;
      dweight[cc] = accumulate ? (float)((double)dweight[cc] + t2) : (float)t2;
    }
    __syncthreads();
  }
}

// grid (row chunks, C/32).  GP 0: no g' output, 1: gp = g', 2: gp += g'
template <bool MASK, int GP>
__global__ void __launch_bounds__(BN_THREADS) k_bn_bwd_apply(const uint8_t *__restrict__ y, const uint8_t *__restrict__ gr,
                                                             const uint8_t *__restrict__ z, int64_t n, int c,
                                                             const float *__restrict__ mean, const float *__restrict__ invstd,
                                                             const float *__restrict__ weight, const float *__restrict__ sums,
                                                             uint8_t *__restrict__ dz, uint8_t *__restrict__ gp_out) {
  const int q = threadIdx.x & 7, g = blockIdx.y;
  const int ch = g * 32 + 4 * q;
  const int64_t row_bytes = (int64_t)c * 4;
  const float inv_n = (float)(1.0 / (double)n);
  float mu[4], is[4], a[4], b[4], k2[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    mu[j] = __ldg(mean + ch + j);
    is[j] = __ldg(invstd + ch + j);
    a[j] = __ldg(weight + ch + j) * is[j];
    b[j] = __ldg(sums + ch + j) * inv_n;
    k2[j] = __ldg(sums + c + ch + j) * inv_n;
  }
  for (int64_t r = (int64_t)blockIdx.x * BN_ROW_SLOTS + (threadIdx.x >> 3); r < n; r += (int64_t)gridDim.x * BN_ROW_SLOTS) {
    const int64_t off = r * row_bytes + (int64_t)g * 128;
    float gv[4], zv[4], yv[4], pv[4];
    load4(gr + off, q, gv);
    load4(z + off, q, zv);
    if (MASK) load4(y + off, q, yv);
    if (GP == 2) load4(gp_out + off, q, pv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gp = (MASK && yv[j] <= 0.f) ? 0.f : gv[j];
      const float xh = (zv[j] - mu[j]) * is[j];
      if (GP == 1) pv[j] = gp;
      if (GP == 2) pv[j] += gp;
      gv[j] = a[j] * (gp - b[j] - xh * k2[j]);
    }
    store4(dz + off, q, gv);
    if (GP) store4(gp_out + off, q, pv);
  }
}

template <bool MASK, int GP>
static void launch_bwd_apply(dim3 grid, cudaStream_t st, const void *y, const void *g, const void *z, int64_t n, int c,
                             const float *mean, const float *invstd, const float *weight, const float *sums, void *dz, void *gp) {
  k_bn_bwd_apply<MASK, GP><<<grid, BN_THREADS, 0, st>>>((const uint8_t *)y, (const uint8_t *)g, (const uint8_t *)z, n, c, mean,
                                                        invstd, weight, sums, (uint8_t *)dz, (uint8_t *)gp);
}

static dim3 apply_grid(int64_t n, int c) {
  return dim3((unsigned)std::min<int64_t>(ceil_div(n, BN_ROW_SLOTS), std::max(1, 132 * 8 / (c / 32))), (unsigned)(c / 32));
}

static bool overlaps(const void *a, const void *b, int64_t bytes) {
  if (!a || !b) return false;
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + (uintptr_t)bytes && y < x + (uintptr_t)bytes;
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_bn_stats_workspace_bytes(int64_t n, int32_t c) {
  if (n < 2 || c <= 0 || c % 32 != 0) return 0;
  return (size_t)bn_row_blocks(n) * 2 * (size_t)c * sizeof(double);
}

static int bn_batch_stats(const void *x_split, int64_t n, int32_t c, const float *weight, const float *bias, double eps,
                          double momentum, float *running_mean, float *running_var, int64_t *num_batches_tracked, float *scale,
                          float *shift, float *mean_out, float *invstd_out, void *ws, size_t ws_bytes, void *stream_) {
  OSB_CHECK(n >= 2, "osb_bn_batch_stats: expected more than 1 value per channel when training (n=%lld)", (long long)n);
  OSB_CHECK(c > 0 && c % 32 == 0 && c / 32 <= 65535, "osb_bn_batch_stats: channels (%d) must be a positive multiple of 32", c);
  OSB_CHECK(x_split && weight && bias && running_mean && running_var && num_batches_tracked && scale && shift,
            "osb_bn_batch_stats: null rows, affine parameters, running buffers or outputs");
  OSB_CHECK(eps >= 0.0, "osb_bn_batch_stats: eps (%g) must be non-negative", eps);
  OSB_CHECK(((uintptr_t)x_split & 15) == 0, "osb_bn_batch_stats: rows must be 16-byte aligned");
  const size_t need = osb_bn_stats_workspace_bytes(n, c);
  OSB_CHECK(ws != nullptr && ws_bytes >= need, "osb_bn_batch_stats: workspace of %zu bytes required (got %zu)", need, ws_bytes);
  cudaStream_t stream = (cudaStream_t)stream_;
  const int64_t nblk = bn_row_blocks(n);
  k_bn_partial<<<dim3((unsigned)nblk, (unsigned)(c / 32)), BN_THREADS, 0, stream>>>((const uint8_t *)x_split, n, c, (double *)ws);
  OSB_LAUNCH_CHECK();
  k_bn_finalize<<<1, BN_THREADS, 0, stream>>>((const uint8_t *)x_split, n, c, nblk, (const double *)ws, weight, bias, eps, momentum,
                                              running_mean, running_var, num_batches_tracked, scale, shift, mean_out, invstd_out);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_bn_batch_stats(const void *x_split, int64_t n, int32_t c, const float *weight, const float *bias, double eps,
                       double momentum, float *running_mean, float *running_var, int64_t *num_batches_tracked, float *scale,
                       float *shift, void *ws, size_t ws_bytes, void *stream) {
  return bn_batch_stats(x_split, n, c, weight, bias, eps, momentum, running_mean, running_var, num_batches_tracked, scale, shift,
                        nullptr, nullptr, ws, ws_bytes, stream);
}

int osb_bn_batch_stats_save(const void *x_split, int64_t n, int32_t c, const float *weight, const float *bias, double eps,
                            double momentum, float *running_mean, float *running_var, int64_t *num_batches_tracked, float *scale,
                            float *shift, float *mean, float *invstd, void *ws, size_t ws_bytes, void *stream) {
  OSB_CHECK(mean && invstd, "osb_bn_batch_stats_save: null mean or invstd");
  return bn_batch_stats(x_split, n, c, weight, bias, eps, momentum, running_mean, running_var, num_batches_tracked, scale, shift,
                        mean, invstd, ws, ws_bytes, stream);
}

static int bn_apply(const char *fn, const void *x_split, void *y_split, int64_t n, int32_t c, const float *scale, const float *shift,
                    const void *res_split, const float *res_scale, const float *res_shift, int32_t relu, void *stream_) {
  OSB_CHECK(n >= 2, "%s: expected more than 1 value per channel when training (n=%lld)", fn, (long long)n);
  OSB_CHECK(c > 0 && c % 32 == 0 && c / 32 <= 65535, "%s: channels (%d) must be a positive multiple of 32", fn, c);
  OSB_CHECK(x_split && y_split && scale && shift, "%s: null rows, scale or shift", fn);
  OSB_CHECK((res_scale == nullptr) == (res_shift == nullptr), "%s: res_scale and res_shift go together", fn);
  OSB_CHECK(res_split != nullptr || res_scale == nullptr, "%s: res_scale / res_shift without res_split", fn);
  OSB_CHECK(!overlaps(res_split, x_split, n * 4 * c) && !overlaps(res_split, y_split, n * 4 * c),
            "%s: the residual must not alias the rows", fn);
  OSB_CHECK(x_split == y_split || !overlaps(x_split, y_split, n * 4 * c), "%s: input and output rows overlap", fn);
  OSB_CHECK((((uintptr_t)x_split | (uintptr_t)y_split | (uintptr_t)res_split) & 15) == 0, "%s: rows must be 16-byte aligned", fn);
  cudaStream_t stream = (cudaStream_t)stream_;
  const dim3 grid = apply_grid(n, c);
  const int mode = res_split == nullptr ? 0 : (res_scale == nullptr ? 1 : 2);
  auto go = [&](auto f) { f(grid, stream, x_split, y_split, n, c, scale, shift, res_split, res_scale, res_shift); };
  if (relu) {
    if (mode == 0) go(launch_apply<0, true>); else if (mode == 1) go(launch_apply<1, true>); else go(launch_apply<2, true>);
  } else {
    if (mode == 0) go(launch_apply<0, false>); else if (mode == 1) go(launch_apply<1, false>); else go(launch_apply<2, false>);
  }
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_bn_apply_split(void *x_split, int64_t n, int32_t c, const float *scale, const float *shift, const void *res_split,
                       const float *res_scale, const float *res_shift, int32_t relu, void *stream) {
  return bn_apply("osb_bn_apply_split", x_split, x_split, n, c, scale, shift, res_split, res_scale, res_shift, relu, stream);
}

int osb_bn_apply_split_out(const void *x_split, void *y_split, int64_t n, int32_t c, const float *scale, const float *shift,
                           const void *res_split, const float *res_scale, const float *res_shift, int32_t relu, void *stream) {
  OSB_CHECK(x_split != y_split, "osb_bn_apply_split_out: the output must not be the input (osb_bn_apply_split works in place)");
  return bn_apply("osb_bn_apply_split_out", x_split, y_split, n, c, scale, shift, res_split, res_scale, res_shift, relu, stream);
}

static int bn_bwd_check(const char *fn, const void *y, const void *g, const void *z, int64_t n, int32_t c, const float *mean,
                        const float *invstd) {
  OSB_CHECK(n >= 2, "%s: expected more than 1 value per channel when training (n=%lld)", fn, (long long)n);
  OSB_CHECK(c > 0 && c % 32 == 0 && c / 32 <= 65535, "%s: channels (%d) must be a positive multiple of 32", fn, c);
  OSB_CHECK(g && z && mean && invstd, "%s: null gradient, raw rows, mean or invstd", fn);
  OSB_CHECK((((uintptr_t)y | (uintptr_t)g | (uintptr_t)z) & 15) == 0, "%s: rows must be 16-byte aligned", fn);
  return 0;
}

int osb_bn_backward_reduce(const void *y_split, const void *g_split, const void *z_split, int64_t n, int32_t c, const float *mean,
                           const float *invstd, float *sums, float *dweight, float *dbias, int32_t accumulate, void *ws,
                           size_t ws_bytes, void *stream_) {
  if (bn_bwd_check("osb_bn_backward_reduce", y_split, g_split, z_split, n, c, mean, invstd)) return 1;
  OSB_CHECK(sums && dweight && dbias, "osb_bn_backward_reduce: null sums, dweight or dbias");
  const size_t need = osb_bn_stats_workspace_bytes(n, c);
  OSB_CHECK(ws != nullptr && ws_bytes >= need, "osb_bn_backward_reduce: workspace of %zu bytes required (got %zu)", need, ws_bytes);
  cudaStream_t stream = (cudaStream_t)stream_;
  const int64_t nblk = bn_row_blocks(n);
  const dim3 grid((unsigned)nblk, (unsigned)(c / 32));
  if (y_split)
    k_bn_bwd_partial<true><<<grid, BN_THREADS, 0, stream>>>((const uint8_t *)y_split, (const uint8_t *)g_split,
                                                            (const uint8_t *)z_split, n, c, mean, invstd, (double *)ws);
  else
    k_bn_bwd_partial<false><<<grid, BN_THREADS, 0, stream>>>(nullptr, (const uint8_t *)g_split, (const uint8_t *)z_split, n, c,
                                                             mean, invstd, (double *)ws);
  OSB_LAUNCH_CHECK();
  k_bn_bwd_finalize<<<1, BN_THREADS, 0, stream>>>(c, nblk, (const double *)ws, sums, dweight, dbias, accumulate ? 1 : 0);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_bn_backward_apply(const void *y_split, const void *g_split, const void *z_split, int64_t n, int32_t c, const float *mean,
                          const float *invstd, const float *weight, const float *sums, void *dz_split, void *gp_split,
                          int32_t gp_accumulate, void *stream_) {
  if (bn_bwd_check("osb_bn_backward_apply", y_split, g_split, z_split, n, c, mean, invstd)) return 1;
  OSB_CHECK(weight && sums && dz_split, "osb_bn_backward_apply: null weight, sums or dz");
  OSB_CHECK(gp_split != nullptr || !gp_accumulate, "osb_bn_backward_apply: gp_accumulate without gp_split");
  OSB_CHECK((((uintptr_t)dz_split | (uintptr_t)gp_split) & 15) == 0, "osb_bn_backward_apply: rows must be 16-byte aligned");
  const int64_t bytes = n * 4 * c;
  for (const void *in : {y_split, g_split, z_split})
    OSB_CHECK(!overlaps(dz_split, in, bytes) && !overlaps(gp_split, in, bytes),
              "osb_bn_backward_apply: dz / gp must not alias y, g or z");
  OSB_CHECK(!overlaps(dz_split, gp_split, bytes), "osb_bn_backward_apply: dz and gp overlap");
  cudaStream_t stream = (cudaStream_t)stream_;
  const dim3 grid = apply_grid(n, c);
  const int gp = gp_split == nullptr ? 0 : (gp_accumulate ? 2 : 1);
  auto go = [&](auto f) { f(grid, stream, y_split, g_split, z_split, n, c, mean, invstd, weight, sums, dz_split, gp_split); };
  if (y_split) {
    if (gp == 0) go(launch_bwd_apply<true, 0>); else if (gp == 1) go(launch_bwd_apply<true, 1>); else go(launch_bwd_apply<true, 2>);
  } else {
    if (gp == 0) go(launch_bwd_apply<false, 0>); else if (gp == 1) go(launch_bwd_apply<false, 1>); else go(launch_bwd_apply<false, 2>);
  }
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
