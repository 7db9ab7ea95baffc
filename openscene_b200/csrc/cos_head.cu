// Cosine distillation head on split rows: the last layer of the 3D network (a 1x1x1 convolution cin -> C, C = 512 or 768)
// followed by run/distill.py's loss, mean over the supervised rows of 1 - CosineSimilarity(dim=1, eps=1e-8)(f, t) against the
// fp16 2D features t.  The C-wide rows f = x W and their gradient never go to memory.
//
//   osb_cos_head_fwd  per supervised row r (internal row rows[r]): f = x W (fp32, k ascending), then in fp64
//                     |f|^2 = sum f_j^2, f.t, |t|^2 over the fp32 f and the fp16 t widened exactly; state[r] = (|f|, f.t, |t|);
//                     loss = sum_r (1 - f.t / (max(|f|, eps) max(|t|, eps))) / m (fp64, per-block partials in a fixed order).
//   osb_cos_head_bwd  with g read on the device: dloss/df_r = a_r t_r + b_r f_r,
//                       a_r = -g / (m n1c n2c),   b_r = g (f.t) / (m n1c^2 n2c n1)  (b_r = 0 when n1 = 0),
//                     n1c = max(|f|, eps), n2c = max(|t|, eps): torch 2.11's cosine_similarity, whose clamps run under
//                     no_grad; then, re-associated so that f is never formed again,
//                       dx_r = a_r (t_r W^T) + b_r (x_r G),         G = W W^T                      [cin, cin]
//                       dW   = X^T diag(a) T + (X^T diag(b) X) W                                   [cin, C]
//                     dx is written as split rows at rows[r]; every other row of dx is 0.
//
// Why re-associate instead of recomputing f per tile: recomputing f costs a third product of the full row width (x W, then
// d W^T and x^T d), where the re-associated form has two (T W^T and X^T diag(a) T) plus cin x cin terms that are 8x (cin = 96,
// C = 768) smaller, and its per-row state is two scalars.  The price is conditioning on rows where x W cancels: b_r (x_r G)
// carries error relative to |x||W| rather than |f|.  For the trunk outputs this head sees, |f| is not small against |x||W|,
// and the tests pin the rows where it is (|f| < eps) with operands that do not cancel.
//
// Why CUDA cores and not wgmma: at cin = 96, C = 768 a supervised row costs 2 * 96 * 768 = 147 kFLOP per product against
// 384 B of split row plus 1.5 KB of target, ~70 FLOP/B: above the fp32 ridge (67 TFLOP/s over 3.35 TB/s = 20 FLOP/B), so
// this head is compute-bound on CUDA cores.  Three products (forward; T W^T and X^T diag(a) T backward) are 0.44 MFLOP per
// row: 8.8 GFLOP for 20,000 rows, 71 GFLOP for 160,000.  Measured on an H100 80GB HBM3 at 700 W (scripts/bench_distill_head.py,
// INTEGRATION.md "Cosine head"), forward and backward take 0.62 ms (14 TFLOP/s) and 3.3 ms (21 TFLOP/s), against 1.7 ms and
// 8.3 ms for the tensor-core head launch plus torch's loss chain it replaces, and are 1.8 % and 5.1 % of the step.  A
// split-bf16 wgmma head could cut that share further, but not below what the trunk's step-to-step spread already hides;
// fp32 FMA also keeps f free of the bf16x3 split of W and T.
//
// Tiling (256 threads, 4 x 4 outputs per thread in the products, operands staged in shared memory as fp32).  ptxas for
// sm_90a: no spills; k_cos_head_fwd 79 registers and 113 KB of dynamic shared memory at cin = 384 (28 KB at 96),
// k_cos_head_dx 61 registers / 21 KB, k_cos_head_dw 40 / 21 KB, every other kernel at most 44 registers.
//   k_cos_head_fwd  64 supervised rows per tile, the tile's x rows in shared memory [cin][64] for the whole tile; the C
//                   columns in 64-wide tiles, W staged in 32 x 64 chunks.  The row sums are reduced across the 16 threads
//                   sharing a row with a fixed shuffle tree; k_cos_head_rows takes the norms and the loss terms and
//                   k_cos_head_loss merges the block partials.
//   k_cos_head_ab   (a, b) per row; k_cos_head_gram G = W W^T.
//   k_cos_head_dx   grid (cin / 32 lines, 128-row tiles): P = T W^T over C and Q = X G over cin, both in 32-deep chunks.
//   k_cos_head_dw   grid (128-column tiles of [T | X], cin / 32 lines, row splits): partial[s] = X^T [diag(a) T | diag(b) X]
//                   over the rows of split s in 32-row chunks; k_cos_head_dw_sum merges the splits in fp64 in order and
//                   k_cos_head_dw_out adds H W (H the X part) in fp64.
// Every assignment of rows to blocks and every merge order is a function of (m, cin, C) only: two calls give identical bits.
#include "common.cuh"
#include "head_tile.cuh"
#include <algorithm>
#include <math.h>

namespace osb {

constexpr int COS_THREADS = 256;
constexpr int COS_MAX_CIN = 384;
constexpr int COS_FWD_BM = 64;                    // rows per forward tile
constexpr int COS_FWD_LD = COS_FWD_BM + 4;        // x tile [cin][COS_FWD_LD]
constexpr int COS_DX_BM = 128;                    // rows per dx tile
constexpr int COS_DX_LD = COS_DX_BM + 4;
constexpr int COS_DW_BN = 128;                    // columns of [T | X] per dW tile
constexpr int64_t COS_MAX_ROW_BLOCKS = 512;
constexpr int64_t COS_MAX_SPLITS = 64;
constexpr double COS_EPS = 1e-8;                  // torch.nn.CosineSimilarity's default

static bool cos_shape_ok(int64_t m, int32_t cin, int32_t c) {
  return m >= 1 && cin >= 32 && cin <= COS_MAX_CIN && cin % 32 == 0 && (c == 512 || c == 768);
}
static int64_t cos_tile_blocks(int64_t m) { return std::min<int64_t>(ceil_div(m, COS_FWD_BM), 1024); }
static int64_t cos_row_blocks(int64_t m) { return std::min<int64_t>(ceil_div(m, COS_THREADS), COS_MAX_ROW_BLOCKS); }
static int64_t cos_splits(int64_t m) { return std::min<int64_t>(ceil_div(m, 512), COS_MAX_SPLITS); }
static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
static size_t cos_fwd_smem(int cin) { return (size_t)cin * COS_FWD_LD * 4 + 32 * 64 * 4; }

// workspace: loss partials [row blocks] fp64 | (a, b) [m] fp32 | G [cin][cin] fp32 | dW partials [splits][cin][C + cin] fp32 |
//            merged [cin][C + cin] fp64
struct CosWs {
  double *part;
  float2 *ab;
  float *gram;
  float *dwp;
  double *dsum;
};
static size_t cos_ws_layout(int64_t m, int cin, int c, void *base, CosWs *out) {
  const int w2 = c + cin;
  const size_t s0 = al256((size_t)cos_row_blocks(m) * sizeof(double));
  const size_t s1 = al256((size_t)m * sizeof(float2));
  const size_t s2 = al256((size_t)cin * cin * sizeof(float));
  const size_t s3 = al256((size_t)cos_splits(m) * cin * w2 * sizeof(float));
  const size_t s4 = al256((size_t)cin * w2 * sizeof(double));
  if (out) {
    uint8_t *p = (uint8_t *)base;
    out->part = (double *)p;
    out->ab = (float2 *)(p + s0);
    out->gram = (float *)(p + s0 + s1);
    out->dwp = (float *)(p + s0 + s1 + s2);
    out->dsum = (double *)(p + s0 + s1 + s2 + s3);
  }
  return s0 + s1 + s2 + s3 + s4;
}

// torch's clamp_min: NaN stays NaN
__device__ inline double cos_clamp(double v) { return v < COS_EPS ? COS_EPS : v; }

__device__ inline void cos_load_t8(const __half *t, float v[8]) {
  union { uint4 u; __half h[8]; } x;
  x.u = __ldg(reinterpret_cast<const uint4 *>(t));
#pragma unroll
  for (int j = 0; j < 8; ++j) v[j] = __half2float(x.h[j]);
}

// forward: per 64-row tile, f = x W column tile by column tile, row sums in fp64: state[r] = (|f|^2, f.t, |t|^2)
__global__ void __launch_bounds__(COS_THREADS) k_cos_head_fwd(const uint8_t *__restrict__ x, int cin, const float *__restrict__ w,
                                                              int c, const int32_t *__restrict__ rows, int64_t m,
                                                              const __half *__restrict__ t, double *__restrict__ state) {
  extern __shared__ __align__(16) float cos_sm[];
  float *xs = cos_sm;                                     // [cin][COS_FWD_LD]
  float *ws = xs + cin * COS_FWD_LD;                      // [32][64]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t row_bytes = (int64_t)cin * 4;
  const int units = cin / 8;                              // 8-channel units per row
  for (int64_t i0 = (int64_t)blockIdx.x * COS_FWD_BM; i0 < m; i0 += (int64_t)gridDim.x * COS_FWD_BM) {
    __syncthreads();                                      // the previous tile's xs is consumed
    for (int u = tid; u < COS_FWD_BM * units; u += COS_THREADS) {
      const int r = u / units, q = u - r * units;
      float v[8];
      if (i0 + r < m) {
        head_load8(x + (int64_t)__ldg(rows + i0 + r) * row_bytes + 128 * (q >> 2), q & 3, v);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) xs[(8 * q + j) * COS_FWD_LD + r] = v[j];
    }
    double ff[4] = {0, 0, 0, 0}, ft[4] = {0, 0, 0, 0}, tt[4] = {0, 0, 0, 0};
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
        for (int u = tid; u < 32 * 16; u += COS_THREADS) {
          const int kk = u >> 4, q = u & 15;
          *reinterpret_cast<float4 *>(ws + kk * 64 + 4 * q) =
              __ldg(reinterpret_cast<const float4 *>(w + (int64_t)(k0 + kk) * c + j0 + 4 * q));
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < 32; ++kk)
          head_fma44(acc, *reinterpret_cast<const float4 *>(xs + (k0 + kk) * COS_FWD_LD + 4 * ty),
                    *reinterpret_cast<const float4 *>(ws + kk * 64 + 4 * tx));
      }
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t i = i0 + 4 * ty + e;
        if (i < m) {
          union { uint2 u; __half h[4]; } tv;
          tv.u = __ldg(reinterpret_cast<const uint2 *>(t + i * c + j0 + 4 * tx));
#pragma unroll
          for (int f = 0; f < 4; ++f) {
            const double fv = (double)acc[e][f], tj = (double)__half2float(tv.h[f]);
            ff[e] = fma(fv, fv, ff[e]);
            ft[e] = fma(fv, tj, ft[e]);
            tt[e] = fma(tj, tj, tt[e]);
          }
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 4; ++e) {
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {                   // the 16 threads of a row group: one half warp
        ff[e] += __shfl_xor_sync(0xffffffffu, ff[e], o);
        ft[e] += __shfl_xor_sync(0xffffffffu, ft[e], o);
        tt[e] += __shfl_xor_sync(0xffffffffu, tt[e], o);
      }
    }
    if (tx == 0) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t i = i0 + 4 * ty + e;
        if (i < m) {
          state[3 * i] = ff[e];
          state[3 * i + 1] = ft[e];
          state[3 * i + 2] = tt[e];
        }
      }
    }
  }
}

// state[r] = (|f|^2, f.t, |t|^2) -> (|f|, f.t, |t|); per-block sum of 1 - cos over rows in order (the fp64 square root and
// division stay out of the product kernel, where their slow paths would cost it a stack frame)
__global__ void __launch_bounds__(COS_THREADS) k_cos_head_rows(double *__restrict__ state, int64_t m, double *__restrict__ part) {
  __shared__ double s[COS_THREADS];
  double blk = 0.0;
  for (int64_t base = (int64_t)blockIdx.x * COS_THREADS; base < m; base += (int64_t)gridDim.x * COS_THREADS) {
    const int64_t i = base + threadIdx.x;
    double l = 0.0;
    if (i < m) {
      const double n1 = sqrt(state[3 * i]), ft = state[3 * i + 1], n2 = sqrt(state[3 * i + 2]);
      state[3 * i] = n1;
      state[3 * i + 2] = n2;
      l = 1.0 - ft / (cos_clamp(n1) * cos_clamp(n2));
    }
    __syncthreads();
    s[threadIdx.x] = l;
    __syncthreads();
    if (threadIdx.x == 0)
      for (int r = 0; r < COS_THREADS; ++r) blk += s[r];
  }
  if (threadIdx.x == 0) part[blockIdx.x] = blk;
}

// one block: loss = sum of the block partials (fixed order) / m
__global__ void __launch_bounds__(COS_THREADS) k_cos_head_loss(const double *__restrict__ part, int64_t nblk, int64_t m,
                                                               float *__restrict__ loss) {
  __shared__ double a[COS_THREADS];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < nblk; i += COS_THREADS) s += part[i];
  a[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double v = 0.0;
    for (int i = 0; i < COS_THREADS; ++i) v += a[i];
    *loss = (float)(v / (double)m);
  }
}

// (a_r, b_r) of every supervised row from its state and the upstream gradient
__global__ void k_cos_head_ab(const double *__restrict__ state, int64_t m, const float *__restrict__ g, float2 *__restrict__ ab) {
  const double gm = (double)*g / (double)m;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    const double n1 = state[3 * i], ft = state[3 * i + 1], n2 = state[3 * i + 2];
    const double n1c = cos_clamp(n1), n2c = cos_clamp(n2);
    const double a = -gm / (n1c * n2c);
    const double b = n1 > 0.0 ? gm * ft / (n1c * n1c * n2c * n1) : (n1 == 0.0 ? 0.0 : a);     // NaN row: NaN
    ab[i] = make_float2((float)a, (float)b);
  }
}

// G = W W^T [cin][cin], grid (cin / 32, cin / 32): one 32 x 32 tile per block, j ascending in fp32
__global__ void __launch_bounds__(COS_THREADS) k_cos_head_gram(const float *__restrict__ w, int cin, int c, float *__restrict__ gram) {
  __shared__ float a[32][33], b[32][33];
  const int tid = threadIdx.x, ci = tid & 31, rg = tid >> 5;     // column ci, rows rg + 8 e
  const int k0 = 32 * blockIdx.y, i0 = 32 * blockIdx.x;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int j0 = 0; j0 < c; j0 += 32) {
    __syncthreads();
    for (int u = tid; u < 32 * 32; u += COS_THREADS) {
      const int r = u >> 5, j = u & 31;
      a[r][j] = __ldg(w + (int64_t)(k0 + r) * c + j0 + j);
      b[r][j] = __ldg(w + (int64_t)(i0 + r) * c + j0 + j);
    }
    __syncthreads();
    for (int j = 0; j < 32; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[e] = fmaf(a[rg + 8 * e][j], b[ci][j], acc[e]);
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) gram[(int64_t)(k0 + rg + 8 * e) * cin + i0 + ci] = acc[e];
}

// dx, grid (cin / 32, 128-row tiles): line b of every row of the tile, a (T W^T) + b (X G), written as split rows at rows[r]
__global__ void __launch_bounds__(COS_THREADS) k_cos_head_dx(const uint8_t *__restrict__ x, int cin, const float *__restrict__ w,
                                                             int c, const int32_t *__restrict__ rows, int64_t m,
                                                             const __half *__restrict__ t, const float2 *__restrict__ ab,
                                                             const float *__restrict__ gram, uint8_t *__restrict__ dx) {
  __shared__ __align__(16) float as[32][COS_DX_LD];          // T or X chunk, [depth][row]
  __shared__ __align__(16) float bs[32][32];                 // W^T or G chunk, [depth][channel]
  const int tid = threadIdx.x, tx = tid & 7, ty = tid >> 3;  // channels 4 tx .., rows 4 ty ..
  const int b = blockIdx.x;
  const int64_t i0 = (int64_t)blockIdx.y * COS_DX_BM;
  const int64_t row_bytes = (int64_t)cin * 4;
  float p[4][4], q[4][4];
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int f = 0; f < 4; ++f) p[e][f] = q[e][f] = 0.f;
  for (int j0 = 0; j0 < c; j0 += 32) {                       // P = T W^T
    __syncthreads();
    for (int u = tid; u < COS_DX_BM * 4; u += COS_THREADS) {
      const int r = u >> 2, qq = u & 3;
      float v[8];
      if (i0 + r < m) {
        cos_load_t8(t + (i0 + r) * c + j0 + 8 * qq, v);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) as[8 * qq + j][r] = v[j];
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
  for (int k0 = 0; k0 < cin; k0 += 32) {                     // Q = X G
    __syncthreads();
    for (int u = tid; u < COS_DX_BM * 4; u += COS_THREADS) {
      const int r = u >> 2, qq = u & 3;
      float v[8];
      if (i0 + r < m) {
        head_load8(x + (int64_t)__ldg(rows + i0 + r) * row_bytes + 4 * k0, qq, v);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) as[8 * qq + j][r] = v[j];
    }
    {
      const int kk = tid >> 3, cq = tid & 7;                 // G[k0 + kk][32 b + 4 cq ..]
      *reinterpret_cast<float4 *>(&bs[kk][4 * cq]) =
          __ldg(reinterpret_cast<const float4 *>(gram + (int64_t)(k0 + kk) * cin + 32 * b + 4 * cq));
    }
    __syncthreads();
#pragma unroll 8
    for (int d = 0; d < 32; ++d)
      head_fma44(q, *reinterpret_cast<const float4 *>(&as[d][4 * ty]), *reinterpret_cast<const float4 *>(&bs[d][4 * tx]));
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int64_t i = i0 + 4 * ty + e;
    if (i < m) {
      const float2 s = __ldg(ab + i);
      union { uint2 u; __nv_bfloat16 h[4]; } hi, lo;
#pragma unroll
      for (int f = 0; f < 4; ++f) split_bf16(fmaf(s.x, p[e][f], s.y * q[e][f]), hi.h[f], lo.h[f]);
      uint8_t *line = dx + (int64_t)__ldg(rows + i) * row_bytes + 128 * b;
      *reinterpret_cast<uint2 *>(line + 8 * tx) = hi.u;
      *reinterpret_cast<uint2 *>(line + 64 + 8 * tx) = lo.u;
    }
  }
}

// dW partials, grid (column tiles of [T | X], cin / 32, splits): partial[s][k][col] = sum over the split's rows of
// x[k] * (col < C ? a t[col] : b x[col - C]), rows ascending in fp32
__global__ void __launch_bounds__(COS_THREADS) k_cos_head_dw(const uint8_t *__restrict__ x, int cin, int c,
                                                             const int32_t *__restrict__ rows, int64_t m,
                                                             const __half *__restrict__ t, const float2 *__restrict__ ab,
                                                             float *__restrict__ dwp) {
  __shared__ __align__(16) float xa[32][36];                 // [row][channel of line kb]
  __shared__ __align__(16) float bs[32][COS_DW_BN];          // [row][column]
  const int tid = threadIdx.x, kq = tid & 7, cg = tid >> 3;  // channels 4 kq .., columns 4 cg ..
  const int col0 = COS_DW_BN * blockIdx.x, kb = blockIdx.y, w2 = c + cin;
  const bool tpart = col0 < c;                               // C is a multiple of 128: a tile is all T or all X
  const int64_t rps = (m + gridDim.z - 1) / gridDim.z;
  const int64_t r0 = (int64_t)blockIdx.z * rps, r1 = std::min(m, r0 + rps);
  const int64_t row_bytes = (int64_t)cin * 4;
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
    for (int u = tid; u < 32 * (COS_DW_BN / 8); u += COS_THREADS) {
      const int r = u >> 4, qq = u & 15;
      const int col = col0 + 8 * qq;
      float v[8];
      if (r < nr && col < w2) {
        const int64_t i = base + r;
        const float2 s = __ldg(ab + i);
        if (tpart) {
          cos_load_t8(t + i * c + col, v);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] *= s.x;
        } else {
          const int ch = col - c;
          head_load8(x + (int64_t)__ldg(rows + i) * row_bytes + 128 * (ch >> 5), (ch & 31) >> 3, v);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] *= s.y;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
      *reinterpret_cast<float4 *>(&bs[r][8 * qq]) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4 *>(&bs[r][8 * qq + 4]) = make_float4(v[4], v[5], v[6], v[7]);
    }
    __syncthreads();
    for (int r = 0; r < nr; ++r)
      head_fma44(acc, *reinterpret_cast<const float4 *>(&xa[r][4 * kq]), *reinterpret_cast<const float4 *>(&bs[r][4 * cg]));
  }
  const int col = col0 + 4 * cg;
  if (col < w2) {
#pragma unroll
    for (int e = 0; e < 4; ++e)
      *reinterpret_cast<float4 *>(dwp + ((int64_t)blockIdx.z * cin + 32 * kb + 4 * kq + e) * w2 + col) =
          make_float4(acc[e][0], acc[e][1], acc[e][2], acc[e][3]);
  }
}

// dsum[k][col] = sum over splits, in order, fp64
__global__ void k_cos_head_dw_sum(const float *__restrict__ dwp, int64_t splits, int64_t nel, double *__restrict__ dsum) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nel; i += (int64_t)gridDim.x * blockDim.x) {
    double a = 0.0;
    for (int64_t s = 0; s < splits; ++s) a += (double)dwp[s * nel + i];
    dsum[i] = a;
  }
}

// dW[k][j] = dsum[k][j] + sum_i H[k][i] W[i][j], H = dsum[:, C:], i ascending in fp64
__global__ void k_cos_head_dw_out(const double *__restrict__ dsum, const float *__restrict__ w, int cin, int c, float *__restrict__ dw) {
  const int w2 = c + cin;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < (int64_t)cin * c; e += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(e / c), j = (int)(e - (int64_t)k * c);
    double a = dsum[(int64_t)k * w2 + j];
    for (int i = 0; i < cin; ++i) a = fma(dsum[(int64_t)k * w2 + c + i], (double)__ldg(w + (int64_t)i * c + j), a);
    dw[e] = (float)a;
  }
}

static bool cos_overlaps(const void *a, int64_t abytes, const void *b, int64_t bbytes) {
  if (!a || !b) return false;
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + (uintptr_t)bbytes && y < x + (uintptr_t)abytes;
}

static int cos_check(const char *fn, const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *rows,
                     int64_t m, const void *target, const void *ws, size_t ws_bytes) {
  OSB_CHECK(n >= 1, "%s: rows (%lld) must be positive", fn, (long long)n);
  OSB_CHECK(m >= 1 && m <= n, "%s: supervised rows (%lld) must be 1 to %lld", fn, (long long)m, (long long)n);
  OSB_CHECK(cin >= 32 && cin <= COS_MAX_CIN && cin % 32 == 0, "%s: input channels (%d) must be a multiple of 32 up to %d", fn,
            cin, COS_MAX_CIN);
  OSB_CHECK(c == 512 || c == 768, "%s: output channels (%d) must be 512 or 768", fn, c);
  OSB_CHECK(x_split && w && rows && target, "%s: null rows, weights, row index or target", fn);
  OSB_CHECK(((uintptr_t)x_split & 15) == 0 && ((uintptr_t)w & 15) == 0 && ((uintptr_t)target & 15) == 0,
            "%s: rows, weights and target must be 16-byte aligned", fn);
  const size_t need = cos_ws_layout(m, cin, c, nullptr, nullptr);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 255) == 0,
            "%s: 256-byte aligned workspace of %zu bytes required (got %zu)", fn, need, ws_bytes);
  return 0;
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_cos_head_workspace_bytes(int64_t m, int32_t cin, int32_t c) {
  if (!cos_shape_ok(m, cin, c)) return 0;
  return cos_ws_layout(m, cin, c, nullptr, nullptr);
}

int osb_cos_head_fwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *rows, int64_t m,
                     const void *target, double *state, float *loss, void *ws, size_t ws_bytes, void *stream_) {
  if (cos_check("osb_cos_head_fwd", x_split, n, cin, w, c, rows, m, target, ws, ws_bytes)) return 1;
  OSB_CHECK(state && loss, "osb_cos_head_fwd: null state or loss");
  cudaStream_t stream = (cudaStream_t)stream_;
  CosWs s;
  cos_ws_layout(m, cin, c, ws, &s);
  OSB_SMEM_ATTR_ONCE(k_cos_head_fwd, cos_fwd_smem(COS_MAX_CIN));
  k_cos_head_fwd<<<(unsigned)cos_tile_blocks(m), COS_THREADS, cos_fwd_smem(cin), stream>>>(
      (const uint8_t *)x_split, cin, w, c, rows, m, (const __half *)target, state);
  OSB_LAUNCH_CHECK();
  const int64_t nblk = cos_row_blocks(m);
  k_cos_head_rows<<<(unsigned)nblk, COS_THREADS, 0, stream>>>(state, m, s.part);
  OSB_LAUNCH_CHECK();
  k_cos_head_loss<<<1, COS_THREADS, 0, stream>>>(s.part, nblk, m, loss);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_cos_head_bwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *rows, int64_t m,
                     const void *target, const double *state, const float *g, void *dx_split, float *dw, void *ws,
                     size_t ws_bytes, void *stream_) {
  if (cos_check("osb_cos_head_bwd", x_split, n, cin, w, c, rows, m, target, ws, ws_bytes)) return 1;
  OSB_CHECK(state && g && dx_split && dw, "osb_cos_head_bwd: null state, g, dx or dw");
  OSB_CHECK(((uintptr_t)dx_split & 15) == 0, "osb_cos_head_bwd: dx rows must be 16-byte aligned");
  OSB_CHECK(!cos_overlaps(dx_split, n * 4 * cin, x_split, n * 4 * cin), "osb_cos_head_bwd: dx must not overlap the rows");
  OSB_CHECK(!cos_overlaps(dw, (int64_t)cin * c * 4, ws, (int64_t)ws_bytes), "osb_cos_head_bwd: dw must not overlap the workspace");
  cudaStream_t stream = (cudaStream_t)stream_;
  CosWs s;
  cos_ws_layout(m, cin, c, ws, &s);
  OSB_CUDA(cudaMemsetAsync(dx_split, 0, (size_t)n * 4 * cin, stream));
  k_cos_head_ab<<<(unsigned)std::min<int64_t>(ceil_div(m, 256), 1024), 256, 0, stream>>>(state, m, g, s.ab);
  OSB_LAUNCH_CHECK();
  k_cos_head_gram<<<dim3(cin / 32, cin / 32), COS_THREADS, 0, stream>>>(w, cin, c, s.gram);
  OSB_LAUNCH_CHECK();
  k_cos_head_dx<<<dim3(cin / 32, (unsigned)ceil_div(m, COS_DX_BM)), COS_THREADS, 0, stream>>>(
      (const uint8_t *)x_split, cin, w, c, rows, m, (const __half *)target, s.ab, s.gram, (uint8_t *)dx_split);
  OSB_LAUNCH_CHECK();
  const int64_t splits = cos_splits(m);
  const int w2 = c + cin;
  k_cos_head_dw<<<dim3((unsigned)ceil_div(w2, COS_DW_BN), cin / 32, (unsigned)splits), COS_THREADS, 0, stream>>>(
      (const uint8_t *)x_split, cin, c, rows, m, (const __half *)target, s.ab, s.dwp);
  OSB_LAUNCH_CHECK();
  const int64_t nel = (int64_t)cin * w2;
  k_cos_head_dw_sum<<<(unsigned)ceil_div(nel, 256), 256, 0, stream>>>(s.dwp, splits, nel, s.dsum);
  OSB_LAUNCH_CHECK();
  k_cos_head_dw_out<<<(unsigned)ceil_div((int64_t)cin * c, 256), 256, 0, stream>>>(s.dsum, w, cin, c, dw);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
