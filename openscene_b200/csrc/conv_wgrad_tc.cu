// Weight gradient of the sparse convolution on tensor cores (wgmma) (run/distill.py:333, `loss.backward()` through
// every MinkowskiConvolution / MinkowskiConvolutionTranspose of models/mink_unet.py):
//
//   gW[k][ci][co] = sum_{o : nbr[k][o] >= 0}  x[nbr[k][o], ci] * gout[o, co]
//
// The reduction runs over ROWS, the dimension along which the split-bf16 activations are NOT contiguous: both operands
// are therefore MN-major wgmma operands.  A 128-byte line of a split row, [hi x32 | lo x32] of one 32-channel block, is 64
// consecutive "MN" elements; 8 consecutive rows form the 1024-byte 128B-swizzle atom (physically the same shared-memory
// image the forward kernel gathers, only read with the transpose bits of the instruction set).  Two warpgroups, one per
// input-channel block, multiply 16 rows of their block with 16 rows of up to four output-channel blocks per K step
// (M64 x N64 x K16 each); the fp32 result tile (128 x N<=256) holds, per (block, block) pair, the four products hi*hi, hi*lo,
// lo*hi, lo*lo, which the reduce kernel adds up (the full (hi+lo)(hi+lo) product: slightly MORE accurate than the
// three-term forward).
//
// Work unit = (offset k, pair of input blocks, group of <= 4 output blocks, range of output rows); one CTA per unit writes
// its raw 128 x N accumulator to a partial buffer, a second kernel sums quadrants and row ranges in a fixed order: no
// atomics, bit-reproducible.  Missing neighbours are zero-filled rows of the gathered operand (they add nothing).
#include "tc_ptx.cuh"
#include <algorithm>

namespace osb {

constexpr int WG_THREADS = 384;             // warpgroup 0: row gathers + gout TMA; warpgroups 1, 2: wgmma + epilogue
constexpr int WG_ROWS = 128;                 // rows (the MMA K dimension) per pipeline stage
constexpr int WG_TILE = WG_ROWS * 128;       // one (128 rows x one 32-channel block) tile: 16 KB
constexpr int WG_STAGES = 2;
constexpr int WG_STAGE_BYTES = 6 * WG_TILE;  // 2 input-block tiles + 4 output-block tiles

struct WgradParams {
  const uint8_t *x;            // split rows [n_in, cin]
  const int32_t *nbr;          // [K][n_out] or NULL (identity, K == 1)
  int64_t n_out;
  int K, nbi, nbo;             // input / output channel blocks (cin / 32, cout / 32)
  int n_mt, n_nt, n_rs;        // unit grid: pairs of input blocks, groups of 4 output blocks, row ranges
  int64_t rows_per_rs;         // multiple of WG_ROWS
  float *partial;              // [units][128][256] raw accumulators
};

__global__ void __launch_bounds__(WG_THREADS, 1)
k_conv_wgrad_tc(const __grid_constant__ CUtensorMap tmG, const WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + WG_STAGES * WG_STAGE_BYTES);    // fullA[2], fullB[2], empty[2]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t fullA = smem_u32(bars), fullB = smem_u32(bars + 2), empty0 = smem_u32(bars + 4);

  // unit -> (k, mt, nt, rs)
  int u = blockIdx.x;
  const int rs = u % p.n_rs; u /= p.n_rs;
  const int ntile = u % p.n_nt; u /= p.n_nt;
  const int mt = u % p.n_mt;
  const int k = u / p.n_mt;
  const int ib0 = mt * 2, n_ib = min(2, p.nbi - ib0);          // input blocks of this unit
  const int ob0 = ntile * 4, n_ob = min(4, p.nbo - ob0);       // output blocks
  const int64_t r_begin = (int64_t)rs * p.rows_per_rs, r_end = min(r_begin + p.rows_per_rs, p.n_out);
  const int n_stage = (int)((r_end - r_begin + WG_ROWS - 1) / WG_ROWS);

  if (tid == 0) {
    // fullA: the 128 gathering threads; empty: one arrival per consumer warpgroup
    for (int s = 0; s < WG_STAGES; ++s) { mbar_init(fullA + 8 * s, 128); mbar_init(fullB + 8 * s, 1); mbar_init(empty0 + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid == 32) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmG) : "memory");
  __syncthreads();

  if (warp < 4) {
    // ===== gathered x rows (32 rows per warp and stage, as in the forward kernels); warp 0 also loads the gout tiles =====
    // gout tiles by TMA: rows [r, r+128) x one 32-channel block each (rows past n_out: zero fill)
    const int w = warp, j = lane & 7, q = lane >> 3;
    const int64_t row_bytes = (int64_t)p.nbi * 128;
    int s = 0; uint32_t phase = 0;
    for (int t = 0; t < n_stage; ++t) {
      int32_t ridx[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int64_t o = r_begin + (int64_t)t * WG_ROWS + w * 32 + 4 * i + q;
        ridx[i] = (o < r_end) ? (p.nbr ? __ldg(p.nbr + (int64_t)k * p.n_out + o) : (int32_t)o) : -1;
      }
      mbar_wait(empty0 + 8 * s, phase ^ 1);
      if (warp == 0 && elect_one()) {
        const uint32_t fb = fullB + 8 * s;
        mbar_expect_tx(fb, (uint32_t)(n_ob * WG_TILE));
        const int row = (int)(r_begin + (int64_t)t * WG_ROWS);
        for (int b = 0; b < n_ob; ++b)
          tma_load_2d(smem_u32(smem + s * WG_STAGE_BYTES + (2 + b) * WG_TILE), &tmG, fb, (ob0 + b) * 64, row);
      }
      __syncwarp();
      for (int b = 0; b < 2; ++b) {
        const uint32_t a_dst = smem_u32(smem + s * WG_STAGE_BYTES + b * WG_TILE) + (w * 32 + q) * 128;
        const bool have = b < n_ib;                      // a missing second block is multiplied as zeros (rows 64..127 of D unused)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int m7 = (4 * i + q) & 7;
          const bool valid = have && ridx[i] >= 0;
          const uint8_t *sp = valid ? p.x + (int64_t)ridx[i] * row_bytes + (ib0 + b) * 128 + j * 16 : p.x;
          cp_async16(a_dst + i * 512 + ((j ^ m7) << 4), sp, valid ? 16u : 0u);
        }
      }
      cp_async_arrive_noinc(fullA + 8 * s);
      if (++s == WG_STAGES) { s = 0; phase ^= 1; }
    }
  } else {
    // ===== wgmma: warpgroup g (1, 2) owns input block ib0 + g - 1 = rows [64(g-1), 64g) of the 128 x N accumulator =====
    const int g = (warp >> 2) - 1;
    const bool active = g < n_ib;
    float acc[4 * 32];
#pragma unroll
    for (int i = 0; i < 4 * 32; ++i) acc[i] = 0.f;
    int s = 0; uint32_t phase = 0;
    for (int t = 0; t < n_stage; ++t) {
      mbar_wait(fullB + 8 * s, phase);
      mbar_wait(fullA + 8 * s, phase);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // cp.async (generic proxy) writes -> wgmma reads
      if (active) {
        const uint32_t base = smem_u32(smem + s * WG_STAGE_BYTES);
        const uint64_t da = gmma_desc_mn(base + g * WG_TILE, WG_TILE);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < WG_ROWS / 16; ++ks)          // 16 rows = two 1024-byte atoms per K step
#pragma unroll
          for (int b = 0; b < 4; ++b)
            if (b < n_ob)
              wgmma_n64_bf16<1, 1>(acc + 32 * b, da + (uint64_t)(ks * 128), gmma_desc_mn(base + (2 + b) * WG_TILE, WG_TILE) + (uint64_t)(ks * 128), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_hold(acc);
      }
      if ((tid & 127) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * s) : "memory");
      if (++s == WG_STAGES) { s = 0; phase ^= 1; }
    }
    // ---- epilogue: raw accumulator rows of this warp -> partial[unit] (rows and columns the reduce kernel reads)
    if (active) {
      float *dst = p.partial + (int64_t)blockIdx.x * 128 * 256;
      const int r = 64 * g + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
      for (int b = 0; b < 4; ++b)
        if (b < n_ob)
#pragma unroll
          for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int h = 0; h < 2; ++h)
              *reinterpret_cast<float2 *>(dst + (int64_t)(r + 8 * h) * 256 + 64 * b + 8 * i + cq) =
                  make_float2(acc[32 * b + 4 * i + 2 * h], acc[32 * b + 4 * i + 2 * h + 1]);
    }
  }
}

// gw[k][ci][co] = sum over row ranges and over the four (hi|lo) x (hi|lo) quadrants of the unit's accumulator
__global__ void k_conv_wgrad_reduce(const float *__restrict__ partial, int K, int cin, int cout, int n_mt, int n_nt, int n_rs,
                                    float *__restrict__ gw) {
  const int64_t total = (int64_t)K * cin * cout;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int co = (int)(e % cout);
    const int64_t kc = e / cout;
    const int ci = (int)(kc % cin), k = (int)(kc / cin);
    const int cb = ci >> 5, mt = cb >> 1, row_hi = (cb & 1) * 64 + (ci & 31);
    const int ob = co >> 5, ntile = ob >> 2, col_hi = (ob & 3) * 64 + (co & 31);
    float acc = 0.f;
    for (int rs = 0; rs < n_rs; ++rs) {
      const int64_t unit = (((int64_t)k * n_mt + mt) * n_nt + ntile) * n_rs + rs;
      const float *t = partial + unit * 128 * 256;
      acc += (t[row_hi * 256 + col_hi] + t[row_hi * 256 + col_hi + 32]) + (t[(row_hi + 32) * 256 + col_hi] + t[(row_hi + 32) * 256 + col_hi + 32]);
    }
    gw[e] = acc;
  }
}

}  // namespace osb

using namespace osb;

static void wgrad_plan(int64_t n_out, int K, int cin, int cout, int *n_mt, int *n_nt, int *n_rs, int64_t *rows_per_rs) {
  *n_mt = (cin / 32 + 1) / 2;
  *n_nt = (cout / 32 + 3) / 4;
  const int64_t base = (int64_t)K * *n_mt * *n_nt;
  const int64_t chunks = ceil_div(n_out, WG_ROWS);
  int64_t rs = std::max<int64_t>(1, (2 * 132 + base - 1) / base);           // about two CTAs' worth of units per SM ...
  rs = std::min(rs, std::max<int64_t>(1, chunks / 4));                      // ... but at least 4 stages per unit
  *rows_per_rs = ceil_div(chunks, rs) * WG_ROWS;
  *n_rs = (int)ceil_div(n_out, *rows_per_rs);
}

extern "C" {

size_t osb_conv_wgrad_tc_workspace_bytes(int64_t n_out, int32_t K, int32_t cin, int32_t cout) {
  if (n_out <= 0 || K < 1 || cin < 32 || cout < 32) return 0;     // shapes osb_conv_wgrad_tc rejects: nothing to reserve
  int n_mt, n_nt, n_rs; int64_t rpr;
  wgrad_plan(n_out, K, cin, cout, &n_mt, &n_nt, &n_rs, &rpr);
  return (size_t)K * n_mt * n_nt * n_rs * 128 * 256 * sizeof(float);
}

int osb_conv_wgrad_tc(const void *x_split, int32_t cin, int64_t n_in, const int32_t *nbr, int64_t n_out, int32_t K,
                      const void *gout_split, int32_t cout, float *gw, void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(x_split && gout_split && gw, "osb_conv_wgrad_tc: null argument");
  OSB_CHECK(cin > 0 && cin % 32 == 0 && cout > 0 && cout % 32 == 0, "osb_conv_wgrad_tc: channel counts must be multiples of 32 (%d, %d)", cin, cout);
  OSB_CHECK(K >= 1 && (nbr != nullptr || K == 1), "osb_conv_wgrad_tc: identity map needs K == 1");
  OSB_CHECK(n_out > 0 && n_out < (1ll << 31) && n_in > 0, "osb_conv_wgrad_tc: bad row counts");
  WgradParams p{};
  wgrad_plan(n_out, K, cin, cout, &p.n_mt, &p.n_nt, &p.n_rs, &p.rows_per_rs);
  const size_t need = osb_conv_wgrad_tc_workspace_bytes(n_out, K, cin, cout);
  OSB_CHECK(ws != nullptr && ws_bytes >= need, "osb_conv_wgrad_tc: workspace of %zu bytes required (got %zu)", need, ws_bytes);
  p.x = (const uint8_t *)x_split; p.nbr = nbr; p.n_out = n_out; p.K = K; p.nbi = cin / 32; p.nbo = cout / 32;
  p.partial = (float *)ws;
  CUtensorMap tmG;
  if (make_tmap_2b(&tmG, gout_split, 2ull * cout, (uint64_t)n_out, WG_ROWS, 0)) return 1;
  const size_t smem_bytes = (size_t)WG_STAGES * WG_STAGE_BYTES + 128 + 1024;
  OSB_SMEM_ATTR_ONCE(k_conv_wgrad_tc, 227 * 1024);
  const int64_t units = (int64_t)K * p.n_mt * p.n_nt * p.n_rs;
  k_conv_wgrad_tc<<<(unsigned)units, WG_THREADS, smem_bytes, stream>>>(tmG, p);
  OSB_LAUNCH_CHECK();
  const int64_t total = (int64_t)K * cin * cout;
  k_conv_wgrad_reduce<<<(unsigned)std::min<int64_t>(ceil_div(total, 256), 132 * 8), 256, 0, stream>>>(p.partial, K, cin, cout, p.n_mt, p.n_nt,
                                                                                                     p.n_rs, gw);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
