// Generic fp32 sparse convolution on CUDA cores (any channel count, any kernel map).
//
// This is the shape-agnostic path behind MinkowskiConvolution / MinkowskiConvolutionTranspose
// (models/mink_unet.py:47-113) and their backward (run/distill.py:333): output-stationary
// gather -> FFMA -> single write, no atomics on the forward/dgrad path.  The tcgen05 kernel in
// conv_tc.cu is the fast path for the MinkUNet channel plans; this one covers everything else
// (odd channel counts, training-mode gradients) and serves as the fp32 cross-check for it.
#include "common.cuh"
#include <algorithm>

namespace osb {

constexpr int BM = 64, BN = 64, BK = 16;

// out[o, n0:n0+64] = sum_k sum_c in[nbr[k][o], c] * W[k][c][n]
__global__ void __launch_bounds__(256)
k_conv_fwd_f32(const float *__restrict__ in, int64_t ld_in, const int32_t *__restrict__ nbr, int64_t n_out, int K,
               const float *__restrict__ w, int cin, int cout, int transpose_w, float *__restrict__ out) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ int32_t s_idx[BM];

  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  const int64_t row0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;
  const bool vec_a = ((cin & 3) == 0) && ((ld_in & 3) == 0) && ((reinterpret_cast<uintptr_t>(in) & 15) == 0);

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k = 0; k < K; ++k) {
    __syncthreads();  // previous iteration's readers of s_idx / tiles are done
    int valid = 0;
    if (t < BM) {
      const int64_t o = row0 + t;
      int32_t i = -1;
      if (o < n_out) i = nbr ? nbr[(int64_t)k * n_out + o] : (int32_t)o;
      s_idx[t] = i;
      valid = i >= 0;
    }
    if (!__syncthreads_or(valid)) continue;

    for (int c0 = 0; c0 < cin; c0 += BK) {
      {  // A tile: 64 rows x 16 channels
        const int m = t >> 2, kk4 = (t & 3) * 4;
        const int32_t i = s_idx[m];
        float v[4] = {0.f, 0.f, 0.f, 0.f};
        if (i >= 0) {
          const float *p = in + (int64_t)i * ld_in + c0 + kk4;
          if (vec_a && c0 + kk4 + 3 < cin) {
            const float4 q = __ldg(reinterpret_cast<const float4 *>(p));
            v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j)
              if (c0 + kk4 + j < cin) v[j] = __ldg(p + j);
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) As[kk4 + j][m] = v[j];
      }
      {  // B tile: 16 channels x 64 outputs
        const int kk = t >> 4, n4 = (t & 15) * 4;
        const int c = c0 + kk;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int n = n0 + n4 + j;
          float v = 0.f;
          if (c < cin && n < cout)
            v = transpose_w ? __ldg(w + ((int64_t)k * cout + n) * cin + c) : __ldg(w + ((int64_t)k * cin + c) * cout + n);
          Bs[kk][n4 + j] = v;
        }
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < BK; ++kk) {
        const float4 a = *reinterpret_cast<const float4 *>(&As[kk][ty * 4]);
        const float4 b = *reinterpret_cast<const float4 *>(&Bs[kk][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t o = row0 + ty * 4 + i;
    if (o >= n_out) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < cout) out[o * cout + n] = acc[i][j];
    }
  }
}

// gw[k][ci][co] += sum_{o in chunk} in[nbr[k][o]][ci] * gout[o][co]
constexpr int WG_ROWS = 4096;
__global__ void __launch_bounds__(256)
k_conv_wgrad_f32(const float *__restrict__ in, const int32_t *__restrict__ nbr, int64_t n_out, int K,
                 const float *__restrict__ gout, int cin, int cout, float *__restrict__ gw) {
  __shared__ float As[BK][BM + 4];  // [o][ci]
  __shared__ float Bs[BK][BN + 4];  // [o][co]
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  const int k = blockIdx.z;
  const int tiles_co = (cout + BN - 1) / BN;
  const int ci0 = (blockIdx.y / tiles_co) * BM, co0 = (blockIdx.y % tiles_co) * BN;
  const int64_t o_begin = (int64_t)blockIdx.x * WG_ROWS;
  const int64_t o_end = min(o_begin + (int64_t)WG_ROWS, n_out);

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int64_t ob = o_begin; ob < o_end; ob += BK) {
    {
      const int oo = t >> 4, c4 = (t & 15) * 4;
      const int64_t o = ob + oo;
      int32_t i = -1;
      if (o < o_end) i = nbr ? nbr[(int64_t)k * n_out + o] : (int32_t)o;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int ci = ci0 + c4 + j, co = co0 + c4 + j;
        As[oo][c4 + j] = (i >= 0 && ci < cin) ? __ldg(in + (int64_t)i * cin + ci) : 0.f;
        Bs[oo][c4 + j] = (i >= 0 && co < cout) ? __ldg(gout + o * cout + co) : 0.f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 a = *reinterpret_cast<const float4 *>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4 *>(&Bs[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ci = ci0 + ty * 4 + i;
    if (ci >= cin) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = co0 + tx * 4 + j;
      if (co < cout && acc[i][j] != 0.f) atomicAdd(gw + ((int64_t)k * cin + ci) * cout + co, acc[i][j]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// "Thin" convolutions: cin <= 4, cout == 32 -- the 5x5x5 stem (conv0p1s1, models/mink_unet.py:47-49) in TRAINING, where the
// fused inference stem (conv_stem.cu) does not apply.  The 64x64x16 tiles above waste 13/16 of their K depth on cin = 3 and
// the atomics of the generic wgrad serialise on 125 x 3 x 32 addresses (1.3 ms + 6.2 ms of a 27 ms distillation step on the
// 197k-voxel scene).  Here a lane is an output channel: weights live in shared memory, a warp walks the 125 offsets of its
// row(s) with one coalesced index load per 32 offsets / rows and broadcast loads of the <= 4 input values.
constexpr int THIN_COUT = 32;

template <int CIN>
__global__ void __launch_bounds__(256)
k_conv_fwd_thin(const float *__restrict__ in, const int32_t *__restrict__ nbr, int64_t n_out, int K, const float *__restrict__ w,
                float *__restrict__ out) {
  extern __shared__ float s_w[];                       // [K][CIN][32]
  for (int i = threadIdx.x; i < K * CIN * THIN_COUT; i += blockDim.x) s_w[i] = __ldg(w + i);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  for (int64_t o = (int64_t)blockIdx.x * wpb + warp; o < n_out; o += (int64_t)gridDim.x * wpb) {
    float acc = 0.f;
    for (int k0 = 0; k0 < K; k0 += 32) {
      const int kmine = k0 + lane;
      const int32_t mine = kmine < K ? __ldg(nbr + (int64_t)kmine * n_out + o) : -1;      // 32 offsets of this row at once
      unsigned live = __ballot_sync(0xffffffffu, mine >= 0);
      while (live) {                                                                     // only the offsets that have a neighbour
        const int kk = __ffs(live) - 1;
        live &= live - 1;
        const int32_t idx = __shfl_sync(0xffffffffu, mine, kk);
        const float *x = in + (int64_t)idx * CIN;
        const float *wk = s_w + (k0 + kk) * CIN * THIN_COUT + lane;
#pragma unroll
        for (int c = 0; c < CIN; ++c) acc = fmaf(__ldg(x + c), wk[c * THIN_COUT], acc);
      }
    }
    out[o * THIN_COUT + lane] = acc;
  }
}

// gw[k][ci][lane] += sum_o in[nbr[k][o]][ci] * gout[o][lane].  A warp owns the offsets k = warp, warp + 8, ... (<= 16 of them for
// K = 125) and keeps their CIN accumulators in registers over ALL rows of the block's share; rows are walked 32 at a time (one
// coalesced index load per offset), the output-gradient rows of a chunk are staged in shared memory once for all offsets.
constexpr int THIN_WG_WARPS = 8, THIN_WG_KPW = 16, THIN_WG_ROWS = 128;

template <int CIN>
__global__ void __launch_bounds__(THIN_WG_WARPS * 32)
k_conv_wgrad_thin(const float *__restrict__ in, const int32_t *__restrict__ nbr, int64_t n_out, int K, const float *__restrict__ gout,
                  float *__restrict__ gw) {
  __shared__ float s_g[THIN_WG_ROWS][THIN_COUT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc[THIN_WG_KPW][CIN];
#pragma unroll
  for (int i = 0; i < THIN_WG_KPW; ++i)
#pragma unroll
    for (int c = 0; c < CIN; ++c) acc[i][c] = 0.f;
  const int64_t n_chunks = (n_out + THIN_WG_ROWS - 1) / THIN_WG_ROWS;
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    const int64_t o0 = ch * THIN_WG_ROWS;
    __syncthreads();                                   // the previous chunk's readers are done
    for (int i = threadIdx.x; i < THIN_WG_ROWS * THIN_COUT; i += blockDim.x) {
      const int64_t o = o0 + (i >> 5);
      s_g[i >> 5][i & 31] = o < n_out ? __ldg(gout + o * THIN_COUT + (i & 31)) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < THIN_WG_KPW; ++i) {
      const int k = warp + i * THIN_WG_WARPS;
      if (k >= K) break;                               // warp-uniform
      for (int r0 = 0; r0 < THIN_WG_ROWS; r0 += 32) {
        const int64_t o = o0 + r0 + lane;
        const int32_t mine = o < n_out ? __ldg(nbr + (int64_t)k * n_out + o) : -1;        // 32 rows of this offset at once
        unsigned live = __ballot_sync(0xffffffffu, mine >= 0);
        while (live) {
          const int rr = __ffs(live) - 1;
          live &= live - 1;
          const int32_t idx = __shfl_sync(0xffffffffu, mine, rr);
          const float g = s_g[r0 + rr][lane];
          const float *x = in + (int64_t)idx * CIN;
#pragma unroll
          for (int c = 0; c < CIN; ++c) acc[i][c] = fmaf(__ldg(x + c), g, acc[i][c]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < THIN_WG_KPW; ++i) {
    const int k = warp + i * THIN_WG_WARPS;
    if (k >= K) break;
#pragma unroll
    for (int c = 0; c < CIN; ++c) atomicAdd(gw + ((int64_t)k * CIN + c) * THIN_COUT + lane, acc[i][c]);   // one 128-byte RED per (block, k, c)
  }
}

template <int CIN>
static int launch_fwd_thin(const float *in, const int32_t *nbr, int64_t n_out, int K, const float *w, float *out, cudaStream_t stream) {
  const size_t smem = (size_t)K * CIN * THIN_COUT * sizeof(float);
  OSB_SMEM_ATTR_ONCE(k_conv_fwd_thin<CIN>, 96 * 1024);
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n_out, 8), 132 * 8);
  k_conv_fwd_thin<CIN><<<grid, 256, smem, stream>>>(in, nbr, n_out, K, w, out);
  OSB_LAUNCH_CHECK();
  return 0;
}

template <int CIN>
static int launch_wgrad_thin(const float *in, const int32_t *nbr, int64_t n_out, int K, const float *gout, float *gw, cudaStream_t stream) {
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n_out, THIN_WG_ROWS), 132 * 4);
  k_conv_wgrad_thin<CIN><<<grid, THIN_WG_WARPS * 32, 0, stream>>>(in, nbr, n_out, K, gout, gw);
  OSB_LAUNCH_CHECK();
  return 0;
}

__global__ void k_gather_rows_f32(const float *__restrict__ in, const int32_t *__restrict__ idx, int64_t n_out, int c,
                                  float *__restrict__ out) {
  const int64_t total = n_out * c;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / c;
    const int cc = (int)(e - r * c);
    out[e] = __ldg(in + (int64_t)idx[r] * c + cc);
  }
}

}  // namespace osb

using namespace osb;

extern "C" {

int osb_conv_fwd_f32(const float *in, int64_t ld_in, const int32_t *nbr, int64_t n_out, int32_t K, const float *w,
                     int32_t cin, int32_t cout, int32_t transpose_w, float *out, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n_out > 0 && K >= 1 && cin >= 1 && cout >= 1, "osb_conv_fwd_f32: bad shape");
  OSB_CHECK(nbr != nullptr || K == 1, "osb_conv_fwd_f32: identity map requires K == 1");
  OSB_CHECK(ld_in >= cin, "osb_conv_fwd_f32: ld_in %lld < cin %d", (long long)ld_in, cin);
  OSB_CHECK(in && w && out, "osb_conv_fwd_f32: NULL buffer (in %p, w %p, out %p)", (const void *)in, (const void *)w, (void *)out);
  if (nbr != nullptr && !transpose_w && cout == THIN_COUT && cin >= 1 && cin <= 4 && ld_in == cin && K * cin * THIN_COUT * 4 <= 96 * 1024) {
    switch (cin) {                                     // the 5x5x5 stem in training mode
      case 1: return launch_fwd_thin<1>(in, nbr, n_out, K, w, out, stream);
      case 2: return launch_fwd_thin<2>(in, nbr, n_out, K, w, out, stream);
      case 3: return launch_fwd_thin<3>(in, nbr, n_out, K, w, out, stream);
      default: return launch_fwd_thin<4>(in, nbr, n_out, K, w, out, stream);
    }
  }
  dim3 grid((unsigned)ceil_div(n_out, BM), (unsigned)ceil_div(cout, BN));
  k_conv_fwd_f32<<<grid, 256, 0, stream>>>(in, ld_in, nbr, n_out, K, w, cin, cout, transpose_w, out);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_conv_wgrad_f32(const float *in, const int32_t *nbr, int64_t n_out, int32_t K, const float *gout, int32_t cin,
                       int32_t cout, float *gw, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n_out > 0 && K >= 1 && K <= 65535 && cin >= 1 && cout >= 1, "osb_conv_wgrad_f32: bad shape");
  OSB_CHECK(nbr != nullptr || K == 1, "osb_conv_wgrad_f32: identity map requires K == 1");
  OSB_CHECK(in && gout && gw, "osb_conv_wgrad_f32: NULL buffer (in %p, gout %p, gw %p)", (const void *)in, (const void *)gout, (void *)gw);
  OSB_CUDA(cudaMemsetAsync(gw, 0, sizeof(float) * (size_t)K * cin * cout, stream));
  if (nbr != nullptr && cout == THIN_COUT && cin <= 4 && K <= THIN_WG_WARPS * THIN_WG_KPW) {
    switch (cin) {
      case 1: return launch_wgrad_thin<1>(in, nbr, n_out, K, gout, gw, stream);
      case 2: return launch_wgrad_thin<2>(in, nbr, n_out, K, gout, gw, stream);
      case 3: return launch_wgrad_thin<3>(in, nbr, n_out, K, gout, gw, stream);
      default: return launch_wgrad_thin<4>(in, nbr, n_out, K, gout, gw, stream);
    }
  }
  dim3 grid((unsigned)ceil_div(n_out, WG_ROWS), (unsigned)(ceil_div(cin, BM) * ceil_div(cout, BN)), (unsigned)K);
  k_conv_wgrad_f32<<<grid, 256, 0, stream>>>(in, nbr, n_out, K, gout, cin, cout, gw);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_gather_rows_f32(const float *in, const int32_t *idx, int64_t n_out, int32_t c, float *out, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (n_out == 0) return 0;
  OSB_CHECK(n_out > 0 && c > 0 && in && idx && out, "osb_gather_rows_f32: bad arguments (n_out %lld, c %d)", (long long)n_out, c);
  const int64_t total = n_out * c;
  unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(total, 256), 132 * 16);
  k_gather_rows_f32<<<blocks, 256, 0, stream>>>(in, idx, n_out, c, out);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
