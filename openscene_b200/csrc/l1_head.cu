// L1 distillation head on split rows: the last layer of the 3D network (a 1x1x1 convolution cin -> C, C = 512 or 768)
// followed by run/distill.py's loss_type 'l1', torch.nn.L1Loss()(f, t) = mean over the m x C elements of |f - t|, against the
// fp16 2D features t.  The C-wide rows f = x W and their gradient never go to memory.
//
//   osb_l1_head_fwd  per supervised row r (internal row rows[r]): f = x W (fp32, k ascending), d = fp32(f - t) with t the fp16
//                    target widened exactly; loss = fp32(sum |d| / (m C)), the sum in fp64 with per-block partials merged in a
//                    fixed order (a NaN anywhere makes it NaN, an infinite d inf); signs[r] = the 2-bit code of sign(d) of every
//                    element (below).
//   osb_l1_head_bwd  with g read on the device: dloss/df = s sgn(d), s = fp32(g * fp32(1 / fp32(m C))) (torch's CUDA
//                    MeanBackward0: a tensor divided by a CPU scalar is multiplied by its fp32 reciprocal), then
//                      dx_r = s (sgn_r W^T)          dW = s (X^T Sgn)
//                    where sgn is exactly +1, -1 or 0, so both products are sums of +-W or +-x, scaled once by s.  dx is
//                    written as split rows at rows[r]; every other row of dx is 0.
//
// Sign codes, 2 bits per element, uint32 [m, C / 16]: element j of row r is bits 2 (j % 16) .. 2 (j % 16) + 1 of word
// signs[r][j / 16]; code 0 is sign 0 (d = +-0, or d NaN: torch's sgn is (0 < d) - (d < 0)), 1 is +1, 2 is -1; 3 is never
// written.  The backward reads only the codes, never t: its gradient is exactly the gradient of the loss the forward
// reported, and it needs two row-width products (Sgn W^T and X^T Sgn) where recomputing f would need three.
//
// Why CUDA cores and not wgmma: the cosine head's argument (cos_head.cu) holds unchanged -- the same three row-width
// products per supervised row, ~70 FLOP/B at cin = 96, C = 768, above the fp32 ridge.
//
// Tiling (256 threads, 4 x 4 outputs per thread in the products, operands staged in shared memory as fp32): the cosine
// head's, with the sign codes in place of T.
//   k_l1_head_fwd   64 supervised rows per tile, the tile's x rows in shared memory [cin][64]; the C columns in 64-wide
//                   tiles, W staged in 32 x 64 chunks.  Each thread adds its |d| in fp64 in a fixed order, the block's
//                   threads are merged by a fixed shuffle tree and warp order into one partial per block; k_l1_head_loss
//                   merges the block partials.  The four threads sharing a sign word OR their bytes together by shuffles.
//   k_l1_head_dx    grid (cin / 32 lines, 128-row tiles): Sgn W^T over C in 32-deep chunks, times s, split store.
//   k_l1_head_dw    grid (128-column tiles of C, cin / 32 lines, row splits): partial[s] = X^T Sgn over the rows of split s
//                   in 32-row chunks, fp32; k_l1_head_dw_out merges the splits in fp64 in order and multiplies by s.
// ptxas for sm_90a: no spills, no stack; k_l1_head_fwd 48 registers and 113 KB of dynamic shared memory at cin = 384 (28 KB
// at 96), k_l1_head_dx 48 registers / 20.5 KB, k_l1_head_dw 40 / 20.5 KB, k_l1_head_loss 30, k_l1_head_dw_out 32.
// Every assignment of rows to blocks and every merge order is a function of (m, cin, C) only: two calls give identical bits.
// Nothing is launched with PDL.
#include "common.cuh"
#include "head_tile.cuh"
#include <algorithm>
#include <math.h>

namespace osb {

constexpr int L1_THREADS = 256;
constexpr int L1_MAX_CIN = 384;
constexpr int L1_FWD_BM = 64;                     // rows per forward tile
constexpr int L1_FWD_LD = L1_FWD_BM + 4;          // x tile [cin][L1_FWD_LD]
constexpr int L1_DX_BM = 128;                     // rows per dx tile
constexpr int L1_DX_LD = L1_DX_BM + 4;
constexpr int L1_DW_BN = 128;                     // columns of C per dW tile
constexpr int64_t L1_MAX_SPLITS = 64;

static bool l1_shape_ok(int64_t m, int32_t cin, int32_t c) {
  return m >= 1 && cin >= 32 && cin <= L1_MAX_CIN && cin % 32 == 0 && (c == 512 || c == 768);
}
static int64_t l1_tile_blocks(int64_t m) { return std::min<int64_t>(ceil_div(m, L1_FWD_BM), 1024); }
static int64_t l1_splits(int64_t m) { return std::min<int64_t>(ceil_div(m, 512), L1_MAX_SPLITS); }
static size_t l1_al256(size_t x) { return (x + 255) & ~(size_t)255; }
static size_t l1_fwd_smem(int cin) { return (size_t)cin * L1_FWD_LD * 4 + 32 * 64 * 4; }

// workspace: loss partials [tile blocks] fp64 | dW partials [splits][cin][C] fp32
struct L1Ws {
  double *part;
  float *dwp;
};
static size_t l1_ws_layout(int64_t m, int cin, int c, void *base, L1Ws *out) {
  const size_t s0 = l1_al256((size_t)l1_tile_blocks(m) * sizeof(double));
  const size_t s1 = l1_al256((size_t)l1_splits(m) * cin * c * sizeof(float));
  if (out) {
    uint8_t *p = (uint8_t *)base;
    out->part = (double *)p;
    out->dwp = (float *)(p + s0);
  }
  return s0 + s1;
}

// torch's sgn: (0 < d) - (d < 0); NaN and +-0 give code 0
__device__ inline uint32_t l1_code(float d) { return d > 0.f ? 1u : (d < 0.f ? 2u : 0u); }

// the 16 signs of one code word as fp32 +1 / -1 / 0
__device__ inline void l1_decode16(uint32_t word, float v[16]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const uint32_t q = (word >> (2 * j)) & 3u;
    v[j] = (float)(q & 1u) - (float)(q >> 1);
  }
}

// s = g / (m C) as torch's CUDA kernel forms it: g times the fp32 reciprocal of the fp32 element count
__device__ inline float l1_scale(const float *g, int64_t m, int c) {
  return *g * (1.0f / (float)(m * (int64_t)c));
}

// forward: per 64-row tile, f = x W column tile by column tile; sum |f - t| in fp64, the signs of f - t packed
__global__ void __launch_bounds__(L1_THREADS) k_l1_head_fwd(const uint8_t *__restrict__ x, int cin, const float *__restrict__ w,
                                                            int c, const int32_t *__restrict__ rows, int64_t m,
                                                            const __half *__restrict__ t, uint32_t *__restrict__ signs,
                                                            double *__restrict__ part) {
  extern __shared__ __align__(16) float l1_sm[];
  float *xs = l1_sm;                                      // [cin][L1_FWD_LD]
  float *ws = xs + cin * L1_FWD_LD;                       // [32][64]
  __shared__ double wsum[L1_THREADS / 32];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t row_bytes = (int64_t)cin * 4;
  const int units = cin / 8;                              // 8-channel units per row
  const int words = c / 16;                               // sign words per row
  double acc_l = 0.0;
  for (int64_t i0 = (int64_t)blockIdx.x * L1_FWD_BM; i0 < m; i0 += (int64_t)gridDim.x * L1_FWD_BM) {
    __syncthreads();                                      // the previous tile's xs is consumed
    for (int u = tid; u < L1_FWD_BM * units; u += L1_THREADS) {
      const int r = u / units, q = u - r * units;
      float v[8];
      if (i0 + r < m) {
        head_load8(x + (int64_t)__ldg(rows + i0 + r) * row_bytes + 128 * (q >> 2), q & 3, v);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) xs[(8 * q + j) * L1_FWD_LD + r] = v[j];
    }
#pragma unroll 1
    for (int j0 = 0; j0 < c; j0 += 64) {
      float acc[4][4];
#pragma unroll
      for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int f = 0; f < 4; ++f) acc[e][f] = 0.f;
#pragma unroll 1
      for (int k0 = 0; k0 < cin; k0 += 32) {
        __syncthreads();                                  // ws consumed (first chunk: xs staged)
        for (int u = tid; u < 32 * 16; u += L1_THREADS) {
          const int kk = u >> 4, q = u & 15;
          *reinterpret_cast<float4 *>(ws + kk * 64 + 4 * q) =
              __ldg(reinterpret_cast<const float4 *>(w + (int64_t)(k0 + kk) * c + j0 + 4 * q));
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < 32; ++kk)
          head_fma44(acc, *reinterpret_cast<const float4 *>(xs + (k0 + kk) * L1_FWD_LD + 4 * ty),
                     *reinterpret_cast<const float4 *>(ws + kk * 64 + 4 * tx));
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t i = i0 + 4 * ty + e;
        uint32_t byte = 0;
        if (i < m) {
          union { uint2 u; __half h[4]; } tv;
          tv.u = __ldg(reinterpret_cast<const uint2 *>(t + i * c + j0 + 4 * tx));
#pragma unroll
          for (int f = 0; f < 4; ++f) {
            const float d = acc[e][f] - __half2float(tv.h[f]);
            acc_l += (double)fabsf(d);
            byte |= l1_code(d) << (2 * f);
          }
        }
        // columns j0 + 4 tx .. of row i: byte (tx & 3) of word (j0 + 16 (tx >> 2)) / 16; i is the same for the 4 lanes
        uint32_t word = byte << (8 * (tx & 3));
        word |= __shfl_xor_sync(0xffffffffu, word, 1);
        word |= __shfl_xor_sync(0xffffffffu, word, 2);
        if (i < m && (tx & 3) == 0) signs[i * words + (j0 >> 4) + (tx >> 2)] = word;
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc_l += __shfl_xor_sync(0xffffffffu, acc_l, o);
  if ((tid & 31) == 0) wsum[tid >> 5] = acc_l;
  __syncthreads();
  if (tid == 0) {
    double s = 0.0;
    for (int k = 0; k < L1_THREADS / 32; ++k) s += wsum[k];
    part[blockIdx.x] = s;
  }
}

// one block: loss = fp32(sum of the block partials (fixed order) / (m C))
__global__ void __launch_bounds__(L1_THREADS) k_l1_head_loss(const double *__restrict__ part, int64_t nblk, int64_t m, int c,
                                                             float *__restrict__ loss) {
  __shared__ double a[L1_THREADS];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < nblk; i += L1_THREADS) s += part[i];
  a[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int i = 0; i < L1_THREADS; ++i) v += a[i];
    *loss = (float)(v / ((double)m * (double)c));
  }
}

// dx, grid (cin / 32, 128-row tiles): line b of every row of the tile, s (Sgn W^T), written as split rows at rows[r]
__global__ void __launch_bounds__(L1_THREADS) k_l1_head_dx(int cin, const float *__restrict__ w, int c,
                                                           const int32_t *__restrict__ rows, int64_t m,
                                                           const uint32_t *__restrict__ signs, const float *__restrict__ g,
                                                           uint8_t *__restrict__ dx) {
  __shared__ __align__(16) float as[32][L1_DX_LD];           // Sgn chunk, [depth][row]
  __shared__ __align__(16) float bs[32][32];                 // W^T chunk, [depth][channel]
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;  // channels 4 tx .., rows 4 ty ..
  const int b = blockIdx.x;
  const int64_t i0 = (int64_t)blockIdx.y * L1_DX_BM;
  const int64_t row_bytes = (int64_t)cin * 4;
  const int words = c / 16;
  float p[4][4];
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int f = 0; f < 4; ++f) p[e][f] = 0.f;
  for (int j0 = 0; j0 < c; j0 += 32) {
    __syncthreads();
    {
      const int r = tid >> 1, h = tid & 1;                   // 16 columns j0 + 16 h .. of row i0 + r
      float v[16];
      l1_decode16(i0 + r < m ? __ldg(signs + (i0 + r) * words + (j0 >> 4) + h) : 0u, v);
#pragma unroll
      for (int j = 0; j < 16; ++j) as[16 * h + j][r] = v[j];
    }
    {
      const int ch = tid >> 3, jq = tid & 7;                 // W[32 b + ch][j0 + 4 jq ..]
      const float4 v = __ldg(reinterpret_cast<const float4 *>(w + (int64_t)(32 * b + ch) * c + j0 + 4 * jq));
      bs[4 * jq][ch] = v.x; bs[4 * jq + 1][ch] = v.y; bs[4 * jq + 2][ch] = v.z; bs[4 * jq + 3][ch] = v.w;
    }
    __syncthreads();
#pragma unroll 8
    for (int d = 0; d < 32; ++d)
      head_fma44(p, *reinterpret_cast<const float4 *>(&as[d][4 * ty]), *reinterpret_cast<const float4 *>(&bs[d][4 * tx]));
  }
  const float s = l1_scale(g, m, c);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int64_t i = i0 + 4 * ty + e;
    if (i < m) {
      union { uint2 u; __nv_bfloat16 h[4]; } hi, lo;
#pragma unroll
      for (int f = 0; f < 4; ++f) split_bf16(s * p[e][f], hi.h[f], lo.h[f]);
      uint8_t *line = dx + (int64_t)__ldg(rows + i) * row_bytes + 128 * b;
      *reinterpret_cast<uint2 *>(line + 8 * tx) = hi.u;
      *reinterpret_cast<uint2 *>(line + 64 + 8 * tx) = lo.u;
    }
  }
}

// dW partials, grid (column tiles of C, cin / 32, splits): partial[s][k][j] = sum over the split's rows of x[k] sgn[j], rows
// ascending in fp32
__global__ void __launch_bounds__(L1_THREADS) k_l1_head_dw(const uint8_t *__restrict__ x, int cin, int c,
                                                           const int32_t *__restrict__ rows, int64_t m,
                                                           const uint32_t *__restrict__ signs, float *__restrict__ dwp) {
  __shared__ __align__(16) float xa[32][36];                 // [row][channel of line kb]
  __shared__ __align__(16) float bs[32][L1_DW_BN];           // [row][column]
  const int tid = threadIdx.x, kq = tid & 7, cg = tid >> 3;  // channels 4 kq .., columns 4 cg ..
  const int col0 = L1_DW_BN * blockIdx.x, kb = blockIdx.y;
  const int64_t rps = (m + gridDim.z - 1) / gridDim.z;
  const int64_t r0 = (int64_t)blockIdx.z * rps, r1 = std::min(m, r0 + rps);
  const int64_t row_bytes = (int64_t)cin * 4;
  const int words = c / 16;
  float acc[4][4];
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int f = 0; f < 4; ++f) acc[e][f] = 0.f;
  for (int64_t base = r0; base < r1; base += 32) {
    const int nr = (int)std::min<int64_t>(32, r1 - base);
    __syncthreads();
    if (tid < 128) {
      const int r = tid >> 2, qq = tid & 3;
      float v[8];
      if (r < nr) {
        head_load8(x + (int64_t)__ldg(rows + base + r) * row_bytes + 128 * kb, qq, v);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
      *reinterpret_cast<float4 *>(&xa[r][8 * qq]) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4 *>(&xa[r][8 * qq + 4]) = make_float4(v[4], v[5], v[6], v[7]);
    }
    {
      const int r = tid >> 3, qq = tid & 7;                  // 16 columns col0 + 16 qq .. of row base + r
      float v[16];
      l1_decode16(r < nr ? __ldg(signs + (base + r) * words + (col0 >> 4) + qq) : 0u, v);
#pragma unroll
      for (int j = 0; j < 16; j += 4)
        *reinterpret_cast<float4 *>(&bs[r][16 * qq + j]) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
    }
    __syncthreads();
    for (int r = 0; r < nr; ++r)
      head_fma44(acc, *reinterpret_cast<const float4 *>(&xa[r][4 * kq]), *reinterpret_cast<const float4 *>(&bs[r][4 * cg]));
  }
  const int col = col0 + 4 * cg;
#pragma unroll
  for (int e = 0; e < 4; ++e)
    *reinterpret_cast<float4 *>(dwp + ((int64_t)blockIdx.z * cin + 32 * kb + 4 * kq + e) * c + col) =
        make_float4(acc[e][0], acc[e][1], acc[e][2], acc[e][3]);
}

// dW[k][j] = fp32(s * sum over splits, in order, in fp64)
__global__ void k_l1_head_dw_out(const float *__restrict__ dwp, int64_t splits, int64_t m, int c, int64_t nel,
                                 const float *__restrict__ g, float *__restrict__ dw) {
  const double s = (double)l1_scale(g, m, c);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nel; i += (int64_t)gridDim.x * blockDim.x) {
    double a = 0.0;
    for (int64_t k = 0; k < splits; ++k) a += (double)dwp[k * nel + i];
    dw[i] = (float)(s * a);
  }
}

static bool l1_overlaps(const void *a, int64_t abytes, const void *b, int64_t bbytes) {
  if (!a || !b) return false;
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + (uintptr_t)bbytes && y < x + (uintptr_t)abytes;
}

static int l1_check(const char *fn, const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *rows,
                    int64_t m, const uint32_t *signs, const void *ws, size_t ws_bytes) {
  OSB_CHECK(n >= 1, "%s: rows (%lld) must be positive", fn, (long long)n);
  OSB_CHECK(m >= 1 && m <= n, "%s: supervised rows (%lld) must be 1 to %lld", fn, (long long)m, (long long)n);
  OSB_CHECK(cin >= 32 && cin <= L1_MAX_CIN && cin % 32 == 0, "%s: input channels (%d) must be a multiple of 32 up to %d", fn,
            cin, L1_MAX_CIN);
  OSB_CHECK(c == 512 || c == 768, "%s: output channels (%d) must be 512 or 768", fn, c);
  OSB_CHECK(x_split && w && rows && signs, "%s: null rows, weights, row index or signs", fn);
  OSB_CHECK(((uintptr_t)x_split & 15) == 0 && ((uintptr_t)w & 15) == 0 && ((uintptr_t)signs & 15) == 0,
            "%s: rows, weights and signs must be 16-byte aligned", fn);
  const size_t need = l1_ws_layout(m, cin, c, nullptr, nullptr);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 255) == 0,
            "%s: 256-byte aligned workspace of %zu bytes required (got %zu)", fn, need, ws_bytes);
  return 0;
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_l1_head_workspace_bytes(int64_t m, int32_t cin, int32_t c) {
  if (!l1_shape_ok(m, cin, c)) return 0;
  return l1_ws_layout(m, cin, c, nullptr, nullptr);
}

int osb_l1_head_fwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *rows, int64_t m,
                    const void *target, uint32_t *signs, float *loss, void *ws, size_t ws_bytes, void *stream_) {
  if (l1_check("osb_l1_head_fwd", x_split, n, cin, w, c, rows, m, signs, ws, ws_bytes)) return 1;
  OSB_CHECK(target && loss, "osb_l1_head_fwd: null target or loss");
  OSB_CHECK(((uintptr_t)target & 15) == 0, "osb_l1_head_fwd: target must be 16-byte aligned");
  cudaStream_t stream = (cudaStream_t)stream_;
  L1Ws s;
  l1_ws_layout(m, cin, c, ws, &s);
  OSB_SMEM_ATTR_ONCE(k_l1_head_fwd, l1_fwd_smem(L1_MAX_CIN));
  const int64_t nblk = l1_tile_blocks(m);
  k_l1_head_fwd<<<(unsigned)nblk, L1_THREADS, l1_fwd_smem(cin), stream>>>((const uint8_t *)x_split, cin, w, c, rows, m,
                                                                          (const __half *)target, signs, s.part);
  OSB_LAUNCH_CHECK();
  k_l1_head_loss<<<1, L1_THREADS, 0, stream>>>(s.part, nblk, m, c, loss);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_l1_head_bwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *rows, int64_t m,
                    const uint32_t *signs, const float *g, void *dx_split, float *dw, void *ws, size_t ws_bytes, void *stream_) {
  if (l1_check("osb_l1_head_bwd", x_split, n, cin, w, c, rows, m, signs, ws, ws_bytes)) return 1;
  OSB_CHECK(g && dx_split && dw, "osb_l1_head_bwd: null g, dx or dw");
  OSB_CHECK(((uintptr_t)dx_split & 15) == 0, "osb_l1_head_bwd: dx rows must be 16-byte aligned");
  OSB_CHECK(!l1_overlaps(dx_split, n * 4 * cin, x_split, n * 4 * cin), "osb_l1_head_bwd: dx must not overlap the rows");
  OSB_CHECK(!l1_overlaps(dw, (int64_t)cin * c * 4, ws, (int64_t)ws_bytes), "osb_l1_head_bwd: dw must not overlap the workspace");
  cudaStream_t stream = (cudaStream_t)stream_;
  L1Ws s;
  l1_ws_layout(m, cin, c, ws, &s);
  OSB_CUDA(cudaMemsetAsync(dx_split, 0, (size_t)n * 4 * cin, stream));
  k_l1_head_dx<<<dim3(cin / 32, (unsigned)ceil_div(m, L1_DX_BM)), L1_THREADS, 0, stream>>>(cin, w, c, rows, m, signs, g,
                                                                                          (uint8_t *)dx_split);
  OSB_LAUNCH_CHECK();
  const int64_t splits = l1_splits(m);
  k_l1_head_dw<<<dim3((unsigned)(c / L1_DW_BN), cin / 32, (unsigned)splits), L1_THREADS, 0, stream>>>(
      (const uint8_t *)x_split, cin, c, rows, m, signs, s.dwp);
  OSB_LAUNCH_CHECK();
  const int64_t nel = (int64_t)cin * c;
  k_l1_head_dw_out<<<(unsigned)ceil_div(nel, 256), 256, 0, stream>>>(s.dwp, splits, m, c, nel, g, dw);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
