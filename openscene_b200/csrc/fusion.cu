// Multi-view feature fusion on the device (SURVEY.md 8f rank 2): project every 3-D point into a batch of frames,
// depth-test it, gather the pixel's 768-d fp16 feature and keep a running fp32 sum + hit counter per point.
// Replaces the per-frame CPU loop of scripts/feature_fusion/scannet_openseg.py:74-108 and
// PointCloudToImageMapper.compute_mapping (scripts/feature_fusion/fusion_util.py:102-139).
//
// Two kernels per batch of <= 32 frames:
//   k_fusion_map    thread per (frame, point): fp64 projection with the reference's operation order, round-half-even,
//                   border cut, occlusion test against the depth image; writes pix[f][p] = v*W+u or -1.
//   k_fusion_gather warp per point: lanes read the point's <= 32 pixel ids, ballot -> visible frames; points seen by no
//                   frame of the batch cost 128 B of traffic.  Otherwise the fp32 sum row is loaded ONCE, every visible
//                   frame's feature row (C halves, contiguous in the [F,H,W,C] layout) is added in frame order -- the
//                   same sequence of fp32 additions as the reference's `sum_features[mask] += feat` per frame, so the
//                   result is bit-identical -- and stored once.  HBM traffic per visible (point, frame): 2*C bytes of
//                   feature, plus 8*C bytes of sum read+write per point per batch.
#include "common.cuh"

#include <algorithm>

namespace osb {

struct FrameCam { double w2c[16]; double fx, fy, cx, cy; };

template <typename T>
__global__ void __launch_bounds__(256)
k_fusion_map(const T *__restrict__ pts, int64_t n, const double *__restrict__ w2c, const double *__restrict__ intr,
             const double *__restrict__ depth, int n_frames, int H, int W, int cut, double vis_thres,
             int32_t *__restrict__ pix, int32_t *__restrict__ mapping) {
  const int f = blockIdx.y;
  __shared__ double s_m[20];
  if (threadIdx.x < 16) s_m[threadIdx.x] = w2c[16 * f + threadIdx.x];
  else if (threadIdx.x < 20) s_m[threadIdx.x] = intr[4 * f + threadIdx.x - 16];
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = (double)pts[3 * i], y = (double)pts[3 * i + 1], z = (double)pts[3 * i + 2];
  double p[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    // row r of world_to_camera @ [x,y,z,1]^T: the 4-term dot product as a GEMM micro-kernel accumulates it
    double t = __dmul_rn(s_m[4 * r], x);
    t = fma(s_m[4 * r + 1], y, t);
    t = fma(s_m[4 * r + 2], z, t);
    p[r] = __dadd_rn(t, s_m[4 * r + 3]);
  }
  // fusion_util.py:122-124: (p0 * fx) / p2 + cx, then np.round (half to even) and astype(int)
  const double u_f = rint(__dadd_rn(__ddiv_rn(__dmul_rn(p[0], s_m[16]), p[2]), s_m[18]));
  const double v_f = rint(__dadd_rn(__ddiv_rn(__dmul_rn(p[1], s_m[17]), p[2]), s_m[19]));
  bool inside = false;
  int u = 0, v = 0;
  // non-finite or huge values convert to INT64_MIN on the host, which fails `>= cut_bound`
  if (fabs(u_f) < 1e9 && fabs(v_f) < 1e9) {
    u = (int)u_f; v = (int)v_f;
    inside = u >= cut && v >= cut && u < W - cut && v < H - cut;
  }
  if (inside) {
    if (depth != nullptr) {
      const double d = depth[((int64_t)f * H + v) * W + u];
      inside = fabs(__dsub_rn(d, p[2])) <= __dmul_rn(vis_thres, d);      // fusion_util.py:128-132
    } else {
      inside = p[2] > 0.0;                                                // fusion_util.py:134-135
    }
  }
  pix[(int64_t)f * n + i] = inside ? v * W + u : -1;
  if (mapping != nullptr) {
    int32_t *m = mapping + ((int64_t)f * n + i) * 3;
    m[0] = inside ? v : 0; m[1] = inside ? u : 0; m[2] = inside ? 1 : 0;
  }
}

// one warp per point; C % 8 == 0, C <= 1024: lane owns the 16-byte chunks lane, lane+32, ...
constexpr int FUS_MAX_CH = 4;

__global__ void __launch_bounds__(256)
k_fusion_gather(const int32_t *__restrict__ pix, int64_t n, int n_frames, const __half *__restrict__ feat, int64_t frame_stride,
                int C, float *__restrict__ sum, float *__restrict__ counter) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int n_chunks = C / 8;
  for (int64_t p = warp0; p < n; p += n_warps) {
    const int32_t my_pix = lane < n_frames ? pix[(int64_t)lane * n + p] : -1;
    unsigned vis = __ballot_sync(0xffffffffu, my_pix >= 0);
    if (vis == 0) continue;
    float acc[FUS_MAX_CH][8];
    float *srow = sum + p * C;
#pragma unroll
    for (int j = 0; j < FUS_MAX_CH; ++j) {
      const int ch = lane + 32 * j;
      if (ch < n_chunks) {
        const float4 a = *reinterpret_cast<const float4 *>(srow + ch * 8);
        const float4 b = *reinterpret_cast<const float4 *>(srow + ch * 8 + 4);
        acc[j][0] = a.x; acc[j][1] = a.y; acc[j][2] = a.z; acc[j][3] = a.w;
        acc[j][4] = b.x; acc[j][5] = b.y; acc[j][6] = b.z; acc[j][7] = b.w;
      }
    }
    const int hits = __popc(vis);
    while (vis) {
      const int f = __ffs(vis) - 1;
      vis &= vis - 1;
      const int32_t px = __shfl_sync(0xffffffffu, my_pix, f);
      const __half *frow = feat + (int64_t)f * frame_stride + (int64_t)px * C;
      uint4 q[FUS_MAX_CH];
#pragma unroll
      for (int j = 0; j < FUS_MAX_CH; ++j) {
        const int ch = lane + 32 * j;
        if (ch < n_chunks) q[j] = __ldg(reinterpret_cast<const uint4 *>(frow) + ch);
      }
#pragma unroll
      for (int j = 0; j < FUS_MAX_CH; ++j) {
        const int ch = lane + 32 * j;
        if (ch < n_chunks) {
          const __half2 *h = reinterpret_cast<const __half2 *>(&q[j]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 v = __half22float2(h[e]);
            acc[j][2 * e] = __fadd_rn(acc[j][2 * e], v.x);
            acc[j][2 * e + 1] = __fadd_rn(acc[j][2 * e + 1], v.y);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < FUS_MAX_CH; ++j) {
      const int ch = lane + 32 * j;
      if (ch < n_chunks) {
        *reinterpret_cast<float4 *>(srow + ch * 8) = make_float4(acc[j][0], acc[j][1], acc[j][2], acc[j][3]);
        *reinterpret_cast<float4 *>(srow + ch * 8 + 4) = make_float4(acc[j][4], acc[j][5], acc[j][6], acc[j][7]);
      }
    }
    if (lane == 0) counter[p] += (float)hits;     // +1 per visible frame; exact in fp32 below 2^24 frames
  }
}

// feat_bank = sum / (counter == 0 ? 1e-5 : counter)      (scannet_openseg.py:104-105)
__global__ void __launch_bounds__(256)
k_fusion_finalize(const float *__restrict__ sum, const float *__restrict__ counter, int64_t n, int C, float *__restrict__ out) {
  const int64_t total = n * (int64_t)(C / 4);
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = t / (C / 4);
    float c = counter[p];
    if (c == 0.f) c = 1e-5f;
    const float4 s = reinterpret_cast<const float4 *>(sum)[t];
    reinterpret_cast<float4 *>(out)[t] = make_float4(__fdiv_rn(s.x, c), __fdiv_rn(s.y, c), __fdiv_rn(s.z, c), __fdiv_rn(s.w, c));
  }
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_fusion_workspace_bytes(int64_t n, int32_t n_frames) {
  return (size_t)std::max<int64_t>(n, 1) * (size_t)std::max(n_frames, 1) * sizeof(int32_t) + 256;
}

int osb_fusion_accumulate(const void *points, int32_t points_is_f64, int64_t n, const double *w2c, const double *intr,
                          const double *depth, const void *feat, int32_t n_frames, int32_t H, int32_t W, int32_t C,
                          int32_t cut_bound, double vis_thres, float *sum, float *counter, int32_t *mapping, void *ws,
                          size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n >= 0 && n < (1ll << 31), "osb_fusion_accumulate: n out of range");
  OSB_CHECK(n_frames >= 1 && n_frames <= 32, "osb_fusion_accumulate: 1..32 frames per call (got %d)", n_frames);
  OSB_CHECK(H > 0 && W > 0 && (int64_t)H * W < (1ll << 31), "osb_fusion_accumulate: bad image size %d x %d", H, W);
  OSB_CHECK(C > 0 && C % 8 == 0 && C <= 256 * FUS_MAX_CH, "osb_fusion_accumulate: feature width %d must be a multiple of 8, <= %d", C,
            256 * FUS_MAX_CH);
  OSB_CHECK(ws_bytes >= osb_fusion_workspace_bytes(n, n_frames), "osb_fusion_accumulate: workspace too small");
  OSB_CHECK(points && w2c && intr && ws && (feat || !sum), "osb_fusion_accumulate: null argument");
  if (n == 0) return 0;
  int32_t *pix = reinterpret_cast<int32_t *>(ws);
  const dim3 grid((unsigned)ceil_div(n, 256), (unsigned)n_frames);
  if (points_is_f64)
    k_fusion_map<double><<<grid, 256, 0, stream>>>((const double *)points, n, w2c, intr, depth, n_frames, H, W, cut_bound, vis_thres, pix, mapping);
  else
    k_fusion_map<float><<<grid, 256, 0, stream>>>((const float *)points, n, w2c, intr, depth, n_frames, H, W, cut_bound, vis_thres, pix, mapping);
  OSB_LAUNCH_CHECK();
  if (sum != nullptr) {     // mapping-only calls pass sum == nullptr
    OSB_CHECK(counter != nullptr, "osb_fusion_accumulate: counter is null");
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(n, 8), 132 * 16);
    k_fusion_gather<<<blocks, 256, 0, stream>>>(pix, n, n_frames, (const __half *)feat, (int64_t)H * W * C, C, sum, counter);
    OSB_LAUNCH_CHECK();
  }
  return 0;
}

int osb_fusion_finalize(const float *sum, const float *counter, int64_t n, int32_t C, float *feat_bank, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(C > 0 && C % 4 == 0, "osb_fusion_finalize: feature width %d must be a multiple of 4", C);
  if (n == 0) return 0;
  const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(n * (C / 4), 256), 132 * 16);
  k_fusion_finalize<<<blocks, 256, 0, stream>>>(sum, counter, n, C, feat_bank);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
