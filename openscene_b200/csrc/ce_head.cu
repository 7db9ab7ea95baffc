// Softmax cross-entropy head on split rows: the last layer of a per-voxel classifier (a 1x1x1 convolution cin -> C, C small)
// followed by CrossEntropyLoss(ignore_index) with the mean over labelled rows and the argmax the training mIoU needs
// (run/train_mink.py's step).  The logits never go to memory.
//
//   osb_ce_head_fwd  per row: z = x W (fp32), lse = log sum exp z, pred = first argmax (first NaN), nll = lse - z[label];
//                    loss = sum of nll over labelled rows / n_valid (fp64 sum, per-block partials merged in a fixed order).
//   osb_ce_head_bwd  d = (softmax(z) - onehot(label)) g / n_valid on labelled rows (0 elsewhere), dx = d W^T (split rows),
//                    dW = sum_r x_r^T d_r (fp32 per-split partials, merged in fp64 in a fixed order).
//   osb_ce_head_eval the forward row pass over points (run/train_mink.py's validate()): point p reads the row of its voxel,
//                    loss as above over labelled points, pred[p], intersection / union / target counts (metric.cuh) and
//                    a count of labels outside [0, C); no lse, no logits.
//
// Why CUDA cores and not wgmma: for cin = 96, C = 20 a row is 384 B of split bf16 and 2 * 96 * 20 = 3.8 kFLOP of product
// (forward), ~10 FLOP per HBM byte, below the H100's fp32 ridge (67 TFLOP/s over 3.35 TB/s = 20 FLOP/B).  The head is bound
// by reading the rows; tensor cores would only shorten the part that is already hidden, and an N = 24 wgmma with the
// bf16x3 split expansion would need the rows re-laid out as operand tiles.
//
// Row passes (forward, and the first backward kernel) map one row to one lane: the lane reads its row line by line
// (eight 16-byte loads per 128-byte line [hi x32 | lo x32]), keeps 32 logits of one 32-class chunk in registers and reads the
// zero-padded weights W_pad [cin][cp] with warp-uniform float4 loads (one L1 transaction serves the warp).  Softmax state is
// carried across chunks online (running max, rescaled sum), so no lane ever holds more than 32 logits.  No shuffles, no
// cross-lane reductions except the loss partial.
//
// Backward: the row pass writes d [n][C] fp32 to the workspace; a second pass over (row split, 32-channel line) tiles reads
// the x line and d once per tile and produces both dx (that line of every row) and the line's dW partial.  dW needs a
// reduction over rows in a layout (channel x class per thread) that the row pass cannot give without holding cin x C
// accumulators per CTA, which for cin = 384, C = 160 is 240 KB.  Cost: d written and read once more (4 C bytes per row) and
// x read twice, i.e. 384 + 80 + 384 + 80 + 384 + 16 = 1328 B per row for cin = 96, C = 20 (the minimum is 788 B).
//
// Row-to-block assignment and every merge order are functions of n only: two calls give identical bits.
#include "common.cuh"
#include "metric.cuh"
#include <algorithm>
#include <math.h>

namespace osb {

constexpr int CE_THREADS = 256;                     // 8 warps x 32 rows in the row passes
constexpr int CE_MAX_CIN = 384;
constexpr int CE_MAX_C = 160;
constexpr int64_t CE_MAX_ROW_BLOCKS = 1024;
constexpr int CE_TILE = 64;                         // rows per tile of the line pass
constexpr int CE_DS_LD = CE_TILE + 4;               // d tile [cp][CE_DS_LD]: 4 consecutive classes hit 4 different banks
constexpr int64_t CE_MAX_SPLITS = 128;

static bool ce_shape_ok(int64_t n, int32_t cin, int32_t c) {
  return n >= 1 && cin >= 32 && cin <= CE_MAX_CIN && cin % 32 == 0 && c >= 1 && c <= CE_MAX_C;
}
static int ce_cpad(int c) { return (c + 31) / 32 * 32; }
static int64_t ce_row_blocks(int64_t n) { return std::min<int64_t>(ceil_div(n, CE_THREADS), CE_MAX_ROW_BLOCKS); }
static int64_t ce_splits(int64_t n) { return std::min<int64_t>(ceil_div(n, 1024), CE_MAX_SPLITS); }
static size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }
static size_t ce_lines_smem(int cp) { return (size_t)(CE_TILE * 32 + cp * CE_DS_LD + 32 * (cp + 1)) * sizeof(float); }

// workspace: W_pad [cin][cp] | loss partials [row blocks][2] fp64 | d [n][C] fp32 | dW partials [splits][cin][cp] fp32
struct CeWs {
  float *wp;
  double *part;
  float *d;
  float *dwp;
};
static size_t ce_ws_layout(int64_t n, int cin, int c, void *base, CeWs *out) {
  const int cp = ce_cpad(c);
  const size_t a = al256((size_t)cin * cp * sizeof(float));
  const size_t b = al256((size_t)ce_row_blocks(n) * 2 * sizeof(double));
  const size_t d = al256((size_t)n * c * sizeof(float));
  const size_t e = al256((size_t)ce_splits(n) * cin * cp * sizeof(float));
  if (out) {
    uint8_t *p = (uint8_t *)base;
    out->wp = (float *)p;
    out->part = (double *)(p + a);
    out->d = (float *)(p + a + b);
    out->dwp = (float *)(p + a + b + d);
  }
  return a + b + d + e;
}

// evaluation workspace: W_pad [cin][cp] | loss partials [row blocks of n_pts][2] fp64 | labelled points int64 [1]
static size_t ce_eval_ws_layout(int64_t n_pts, int cin, int c, void *base, CeWs *out, int64_t **n_valid) {
  const size_t a = al256((size_t)cin * ce_cpad(c) * sizeof(float));
  const size_t b = al256((size_t)ce_row_blocks(n_pts) * 2 * sizeof(double));
  if (out) {
    uint8_t *p = (uint8_t *)base;
    *out = CeWs{(float *)p, (double *)(p + a), nullptr, nullptr};
    *n_valid = (int64_t *)(p + a + b);
  }
  return a + b + 256;
}

__global__ void k_ce_pad_w(const float *__restrict__ w, int cin, int c, int cp, float *__restrict__ wp) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cin * cp; i += gridDim.x * blockDim.x) {
    const int k = i / cp, j = i - k * cp;
    wp[i] = j < c ? w[k * c + j] : 0.f;
  }
}

// channels 16 h .. 16 h + 15 of a 128-byte line
__device__ inline void ce_load_half(const uint8_t *line, int h, float v[16]) {
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    union { uint4 u; __nv_bfloat16 b[8]; } hi, lo;
    hi.u = __ldg(reinterpret_cast<const uint4 *>(line + 32 * h + 16 * q));
    lo.u = __ldg(reinterpret_cast<const uint4 *>(line + 64 + 32 * h + 16 * q));
#pragma unroll
    for (int j = 0; j < 8; ++j) v[8 * q + j] = join_bf16(hi.b[j], lo.b[j]);
  }
}

// z[c] = x . W_pad[:, 32 j + c], k ascending, fp32
__device__ inline void ce_chunk_logits(const uint8_t *row, int cin, const float *__restrict__ wp, int cp, int j, float z[32]) {
#pragma unroll
  for (int c = 0; c < 32; ++c) z[c] = 0.f;
  for (int b = 0; b < 2 * (cin / 32); ++b) {                    // half lines: 16 channels in registers at a time
    float x[16];
    ce_load_half(row + 128 * (b >> 1), b & 1, x);
    const float *wl = wp + (size_t)(16 * b) * cp + 32 * j;
#pragma unroll
    for (int k = 0; k < 16; ++k) {                               // fully unrolled: x[] stays in registers
      const float4 *w4 = reinterpret_cast<const float4 *>(wl + (size_t)k * cp);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 w = __ldg(w4 + q);
        z[4 * q] = fmaf(x[k], w.x, z[4 * q]);
        z[4 * q + 1] = fmaf(x[k], w.y, z[4 * q + 1]);
        z[4 * q + 2] = fmaf(x[k], w.z, z[4 * q + 2]);
        z[4 * q + 3] = fmaf(x[k], w.w, z[4 * q + 3]);
      }
    }
  }
}

// Evaluation variant of the forward row pass (k_ce_fwd_eval): the pass walks points instead of rows.  Point p reads split
// row row_map[inds_reverse[p]] (row_map[p] without inds_reverse) and its label at p; it writes pred[p] (if pred is set), adds
// its NLL term to the block partial when it is labelled, and counts (pred, label) into the block's shared histogram
// (metric.cuh, intersectionAndUnionGPU's rule), flushed with 64-bit atomics.  A label outside [0, C) other than the ignore
// label leaves the point out of the loss and the counts and is counted in *bad.
struct CeEval {
  const int64_t *inds_reverse;       // NULL: one point per caller row
  uint32_t *hist;                    // shared [3, C]
  unsigned long long *areas;         // [3, C] += intersection | output | target
  int32_t *bad;                      // += points with a label outside [0, C) other than the ignore label
};

// the row pass of k_ce_fwd (EVAL = false: rows in internal order, labels and pred in caller order) and of k_ce_fwd_eval
template <typename L, bool EVAL>
__device__ __forceinline__ void ce_fwd_rows(const uint8_t *__restrict__ x, int64_t n, int cin, const float *__restrict__ wp,
                                            int c, int cp, const int32_t *__restrict__ row_map, const L *__restrict__ labels,
                                            long long ignore, float *__restrict__ lse, int64_t *__restrict__ pred,
                                            double *__restrict__ part, const CeEval ev) {
  __shared__ double s_sum[CE_THREADS / 32], s_cnt[CE_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t row_bytes = (int64_t)cin * 4;
  if constexpr (EVAL) {
    for (int b = threadIdx.x; b < 3 * c; b += CE_THREADS) ev.hist[b] = 0;
    __syncthreads();
  }
  double sum = 0.0, cnt = 0.0;
  for (int64_t grp = (int64_t)blockIdx.x * (CE_THREADS / 32) + warp; grp * 32 < n; grp += (int64_t)gridDim.x * (CE_THREADS / 32)) {
    const int64_t r = grp * 32 + lane;
    const bool valid = r < n;
    const int64_t rr = valid ? r : n - 1;
    int64_t xr = rr;
    int32_t cr = 0;
    long long lab;
    if constexpr (EVAL) {
      xr = __ldg(row_map + (ev.inds_reverse ? __ldg(ev.inds_reverse + rr) : rr));
      lab = (long long)__ldg(labels + rr);
    } else {
      cr = __ldg(row_map + rr);
      lab = (long long)__ldg(labels + cr);
    }
    float m = -INFINITY, s = 0.f, best = -INFINITY, zl = 0.f;
    int arg = 0;
    bool found = false;
    for (int j = 0; j < cp / 32; ++j) {
      float z[32];
      ce_chunk_logits(x + xr * row_bytes, cin, wp, cp, j, z);
      float mc = -INFINITY;
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        const int cc = 32 * j + q;
        if (cc < c) {
          mc = fmaxf(mc, z[q]);
          // strict: the first maximum; a NaN beats everything and is never beaten (torch's max(1)[1]: the first NaN)
          if (z[q] > best || (z[q] != z[q] && best == best)) { best = z[q]; arg = cc; }
          if (cc == lab) { zl = z[q]; found = true; }
        }
      }
      const float mn = fmaxf(m, mc);
      float e = 0.f;
#pragma unroll
      for (int q = 0; q < 32; ++q)
        if (32 * j + q < c) e += expf(z[q] - mn);
      s = s * expf(m - mn) + e;                                  // m = -inf on the first chunk: s = e
      m = mn;
    }
    if (valid) {
      if constexpr (EVAL) {
        if (pred) pred[r] = arg;
        if (lab != ignore && !found) {
          atomicAdd(ev.bad, 1);
        } else {
          if (lab != ignore) {
            sum += (double)(m - zl) + log((double)s);
            cnt += 1.0;
          }
          inter_union_add(arg, lab, c, (int)ignore, ev.hist);
        }
      } else {
        lse[r] = m + logf(s);
        pred[cr] = arg;
        if (lab != ignore) {
          // a label outside [0, C) makes the loss NaN (the caller validates labels first)
          sum += found ? (double)(m - zl) + log((double)s) : (double)NAN;
          cnt += 1.0;
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) { s_sum[warp] = sum; s_cnt[warp] = cnt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int w = 0; w < CE_THREADS / 32; ++w) { a += s_sum[w]; b += s_cnt[w]; }
    part[2 * blockIdx.x] = a;
    part[2 * blockIdx.x + 1] = b;
  }
  if constexpr (EVAL)
    for (int b = threadIdx.x; b < 3 * c; b += CE_THREADS)
      if (ev.hist[b]) atomicAdd(&ev.areas[b], (unsigned long long)ev.hist[b]);
}

// forward row pass: lse, pred (caller order), per-block (sum of nll, labelled rows)
template <typename L>
__global__ void __launch_bounds__(CE_THREADS) k_ce_fwd(const uint8_t *__restrict__ x, int64_t n, int cin,
                                                          const float *__restrict__ wp, int c, int cp,
                                                          const int32_t *__restrict__ row_map, const L *__restrict__ labels,
                                                          long long ignore, float *__restrict__ lse, int64_t *__restrict__ pred,
                                                          double *__restrict__ part) {
  ce_fwd_rows<L, false>(x, n, cin, wp, c, cp, row_map, labels, ignore, lse, pred, part, CeEval{});
}

// evaluation row pass over n_pts points: pred (may be NULL), per-block (sum of nll, labelled points), counts, bad labels
template <typename L>
__global__ void __launch_bounds__(CE_THREADS) k_ce_fwd_eval(const uint8_t *__restrict__ x, int64_t n_pts, int cin,
                                                               const float *__restrict__ wp, int c, int cp,
                                                               const int32_t *__restrict__ row_map,
                                                               const int64_t *__restrict__ inds_reverse,
                                                               const L *__restrict__ labels, int ignore,
                                                               int64_t *__restrict__ pred, double *__restrict__ part,
                                                               unsigned long long *__restrict__ areas, int32_t *__restrict__ bad) {
  __shared__ uint32_t s_hist[3 * CE_MAX_C];
  ce_fwd_rows<L, true>(x, n_pts, cin, wp, c, cp, row_map, labels, ignore, nullptr, pred, part,
                       CeEval{inds_reverse, s_hist, areas, bad});
}

// one block: merge the per-block partials in a fixed order
__global__ void __launch_bounds__(CE_THREADS) k_ce_loss(const double *__restrict__ part, int64_t nblk, float *loss, int64_t *n_valid) {
  __shared__ double a[CE_THREADS], b[CE_THREADS];
  double x = 0.0, y = 0.0;
  for (int64_t i = threadIdx.x; i < nblk; i += CE_THREADS) { x += part[2 * i]; y += part[2 * i + 1]; }
  a[threadIdx.x] = x;
  b[threadIdx.x] = y;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0, c = 0.0;
    for (int i = 0; i < CE_THREADS; ++i) { s += a[i]; c += b[i]; }
    *loss = (float)(s / c);                                      // 0 / 0 = NaN with no labelled row, as torch
    *n_valid = (int64_t)c;
  }
}

// backward row pass: d [n][C] = (softmax(z) - onehot(label)) g / n_valid on labelled rows, else 0 (internal row order)
template <typename L>
__global__ void __launch_bounds__(CE_THREADS) k_ce_bwd_rows(const uint8_t *__restrict__ x, int64_t n, int cin,
                                                               const float *__restrict__ wp, int c, int cp,
                                                               const int32_t *__restrict__ row_map, const L *__restrict__ labels,
                                                               long long ignore, const float *__restrict__ lse,
                                                               const float *__restrict__ g, const int64_t *__restrict__ n_valid,
                                                               float *__restrict__ d) {
  __shared__ float tile[CE_THREADS / 32][32][33];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t row_bytes = (int64_t)cin * 4;
  const int64_t nv = *n_valid;
  const float scale = nv > 0 ? (float)((double)*g / (double)nv) : 0.f;
  for (int64_t grp = (int64_t)blockIdx.x * (CE_THREADS / 32) + warp; grp * 32 < n; grp += (int64_t)gridDim.x * (CE_THREADS / 32)) {
    const int64_t r = grp * 32 + lane;
    const int64_t rr = r < n ? r : n - 1;
    const long long lab = (long long)__ldg(labels + __ldg(row_map + rr));
    const bool labelled = r < n && lab != ignore;
    const float l = __ldg(lse + rr);
    for (int j = 0; j < cp / 32; ++j) {
      float z[32];
      ce_chunk_logits(x + rr * row_bytes, cin, wp, cp, j, z);
#pragma unroll
      for (int q = 0; q < 32; ++q)
        tile[warp][lane][q] = labelled ? (expf(z[q] - l) - (32 * j + q == lab ? 1.f : 0.f)) * scale : 0.f;
      __syncwarp();
      const int cc = 32 * j + lane;
      for (int i = 0; i < 32; ++i) {                             // row i of the group: C consecutive floats
        const int64_t ri = grp * 32 + i;
        if (ri < n && cc < c) d[ri * c + cc] = tile[warp][i][lane];
      }
      __syncwarp();
    }
  }
}

// backward line pass, grid (row splits, cin / 32): for 32-channel line b of every row of the split,
//   dx[r][line b] = d[r] W[line b]^T   and   dW partial[split][line b][:] = sum_r x[r][line b]^T d[r]
__global__ void __launch_bounds__(CE_THREADS) k_ce_bwd_lines(const uint8_t *__restrict__ x, int64_t n, int cin,
                                                             const float *__restrict__ wp, int c, int cp,
                                                             const float *__restrict__ d, uint8_t *__restrict__ dx,
                                                             float *__restrict__ dwp) {
  extern __shared__ __align__(16) float ce_sm[];
  float *xs = ce_sm;                                            // [CE_TILE][32]
  float *ds = xs + CE_TILE * 32;                                // [cp][CE_DS_LD]  (class-major)
  float *wl = ds + cp * CE_DS_LD;                               // [32][cp + 1]
  const int t = threadIdx.x, b = blockIdx.y, nj = cp / 32;
  const int64_t row_bytes = (int64_t)cin * 4;
  const int64_t rpb = (n + gridDim.x - 1) / gridDim.x;
  const int64_t r0 = (int64_t)blockIdx.x * rpb, r1 = std::min(n, r0 + rpb);
  for (int i = t; i < 32 * cp; i += CE_THREADS) {
    const int k = i / cp, j = i - k * cp;
    wl[k * (cp + 1) + j] = wp[(size_t)(32 * b + k) * cp + j];
  }
  const int kq = t & 7, cg = t >> 3;                            // dW: channels 4 kq .. 4 kq + 3, classes cg + 32 i
  const int kx = t & 31, rg = t >> 5;                           // dx: channel kx, rows 8 rg .. 8 rg + 7
  float acc[4][5];
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int i = 0; i < 5; ++i) acc[e][i] = 0.f;
  for (int64_t base = r0; base < r1; base += CE_TILE) {
    const int rows = (int)std::min<int64_t>(CE_TILE, r1 - base);
    __syncthreads();                                            // the previous tile is consumed (first tile: wl staged)
    {
      const int r = t >> 2, q = t & 3;                          // x line: 8 channels per thread
      float v[8];
      if (r < rows) {
        const uint8_t *line = x + (base + r) * row_bytes + 128 * b;
        union { uint4 u; __nv_bfloat16 h[8]; } hi, lo;
        hi.u = __ldg(reinterpret_cast<const uint4 *>(line + 16 * q));
        lo.u = __ldg(reinterpret_cast<const uint4 *>(line + 64 + 16 * q));
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = join_bf16(hi.h[j], lo.h[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
      float4 *o = reinterpret_cast<float4 *>(xs + r * 32 + 8 * q);
      o[0] = make_float4(v[0], v[1], v[2], v[3]);
      o[1] = make_float4(v[4], v[5], v[6], v[7]);
    }
    for (int i = t; i < CE_TILE * cp; i += CE_THREADS) {
      const int r = i / cp, j = i - r * cp;
      ds[j * CE_DS_LD + r] = (r < rows && j < c) ? __ldg(d + (base + r) * c + j) : 0.f;
    }
    __syncthreads();
    for (int r = 0; r < rows; ++r) {
      const float4 xv = *reinterpret_cast<const float4 *>(xs + r * 32 + 4 * kq);
#pragma unroll
      for (int i = 0; i < 5; ++i) {
        if (i < nj) {
          const float dv = ds[(cg + 32 * i) * CE_DS_LD + r];
          acc[0][i] = fmaf(xv.x, dv, acc[0][i]);
          acc[1][i] = fmaf(xv.y, dv, acc[1][i]);
          acc[2][i] = fmaf(xv.z, dv, acc[2][i]);
          acc[3][i] = fmaf(xv.w, dv, acc[3][i]);
        }
      }
    }
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = 0.f;
    for (int j = 0; j < c; ++j) {
      const float w = wl[kx * (cp + 1) + j];
      const float4 d0 = *reinterpret_cast<const float4 *>(ds + j * CE_DS_LD + 8 * rg);
      const float4 d1 = *reinterpret_cast<const float4 *>(ds + j * CE_DS_LD + 8 * rg + 4);
      o[0] = fmaf(d0.x, w, o[0]); o[1] = fmaf(d0.y, w, o[1]); o[2] = fmaf(d0.z, w, o[2]); o[3] = fmaf(d0.w, w, o[3]);
      o[4] = fmaf(d1.x, w, o[4]); o[5] = fmaf(d1.y, w, o[5]); o[6] = fmaf(d1.z, w, o[6]); o[7] = fmaf(d1.w, w, o[7]);
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int r = 8 * rg + i;
      if (r < rows) {
        uint8_t *line = dx + (base + r) * row_bytes + 128 * b;
        __nv_bfloat16 h, l;
        split_bf16(o[i], h, l);
        *reinterpret_cast<__nv_bfloat16 *>(line + 2 * kx) = h;
        *reinterpret_cast<__nv_bfloat16 *>(line + 64 + 2 * kx) = l;
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 4; ++e)
#pragma unroll
    for (int i = 0; i < 5; ++i)
      if (i < nj) dwp[((size_t)blockIdx.x * cin + 32 * b + 4 * kq + e) * cp + cg + 32 * i] = acc[e][i];
}

// dW[k][j] = sum over splits (fixed order, fp64)
__global__ void k_ce_dw_merge(const float *__restrict__ dwp, int64_t splits, int cin, int c, int cp, float *__restrict__ dw) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cin * c; i += gridDim.x * blockDim.x) {
    const int k = i / c, j = i - k * c;
    double a = 0.0;
    for (int64_t s = 0; s < splits; ++s) a += (double)dwp[((size_t)s * cin + k) * cp + j];
    dw[i] = (float)a;
  }
}

static bool ce_overlaps(const void *a, int64_t abytes, const void *b, int64_t bbytes) {
  if (!a || !b) return false;
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + (uintptr_t)bbytes && y < x + (uintptr_t)abytes;
}

static int ce_check(const char *fn, const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *row_map,
                    const void *labels, int32_t labels_are_i64, const void *ws, size_t ws_bytes) {
  OSB_CHECK(n >= 1, "%s: rows (%lld) must be positive", fn, (long long)n);
  OSB_CHECK(cin >= 32 && cin <= CE_MAX_CIN && cin % 32 == 0, "%s: input channels (%d) must be a multiple of 32 up to %d", fn, cin,
            CE_MAX_CIN);
  OSB_CHECK(c >= 1 && c <= CE_MAX_C, "%s: classes (%d) must be 1 to %d", fn, c, CE_MAX_C);
  OSB_CHECK(x_split && w && row_map && labels, "%s: null rows, weights, row map or labels", fn);
  OSB_CHECK(labels_are_i64 == 0 || labels_are_i64 == 1, "%s: labels_are_i64 must be 0 or 1", fn);
  OSB_CHECK(((uintptr_t)x_split & 15) == 0, "%s: rows must be 16-byte aligned", fn);
  const size_t need = ce_ws_layout(n, cin, c, nullptr, nullptr);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 255) == 0,
            "%s: 256-byte aligned workspace of %zu bytes required (got %zu)", fn, need, ws_bytes);
  return 0;
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_ce_head_workspace_bytes(int64_t n, int32_t cin, int32_t c) {
  if (!ce_shape_ok(n, cin, c)) return 0;
  return ce_ws_layout(n, cin, c, nullptr, nullptr);
}

int osb_ce_head_fwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *row_map,
                    const void *labels, int32_t labels_are_i64, int64_t ignore_index, float *lse, int64_t *pred, float *loss,
                    int64_t *n_valid, void *ws, size_t ws_bytes, void *stream_) {
  if (ce_check("osb_ce_head_fwd", x_split, n, cin, w, c, row_map, labels, labels_are_i64, ws, ws_bytes)) return 1;
  OSB_CHECK(lse && pred && loss && n_valid, "osb_ce_head_fwd: null lse, pred, loss or n_valid");
  cudaStream_t stream = (cudaStream_t)stream_;
  CeWs s;
  ce_ws_layout(n, cin, c, ws, &s);
  const int cp = ce_cpad(c);
  k_ce_pad_w<<<(unsigned)ceil_div(cin * cp, 256), 256, 0, stream>>>(w, cin, c, cp, s.wp);
  OSB_LAUNCH_CHECK();
  const int64_t nblk = ce_row_blocks(n);
  if (labels_are_i64)
    k_ce_fwd<int64_t><<<(unsigned)nblk, CE_THREADS, 0, stream>>>((const uint8_t *)x_split, n, cin, s.wp, c, cp, row_map,
                                                                  (const int64_t *)labels, (long long)ignore_index, lse, pred, s.part);
  else
    k_ce_fwd<int32_t><<<(unsigned)nblk, CE_THREADS, 0, stream>>>((const uint8_t *)x_split, n, cin, s.wp, c, cp, row_map,
                                                                  (const int32_t *)labels, (long long)ignore_index, lse, pred, s.part);
  OSB_LAUNCH_CHECK();
  k_ce_loss<<<1, CE_THREADS, 0, stream>>>(s.part, nblk, loss, n_valid);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_ce_head_bwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t c, const int32_t *row_map,
                    const void *labels, int32_t labels_are_i64, int64_t ignore_index, const float *lse, const float *g,
                    const int64_t *n_valid, void *dx_split, float *dw, void *ws, size_t ws_bytes, void *stream_) {
  if (ce_check("osb_ce_head_bwd", x_split, n, cin, w, c, row_map, labels, labels_are_i64, ws, ws_bytes)) return 1;
  OSB_CHECK(lse && g && n_valid && dx_split && dw, "osb_ce_head_bwd: null lse, g, n_valid, dx or dw");
  OSB_CHECK(((uintptr_t)dx_split & 15) == 0, "osb_ce_head_bwd: dx rows must be 16-byte aligned");
  OSB_CHECK(!ce_overlaps(dx_split, n * 4 * cin, x_split, n * 4 * cin), "osb_ce_head_bwd: dx must not overlap the rows");
  OSB_CHECK(!ce_overlaps(dw, (int64_t)cin * c * 4, ws, (int64_t)ws_bytes), "osb_ce_head_bwd: dw must not overlap the workspace");
  cudaStream_t stream = (cudaStream_t)stream_;
  CeWs s;
  ce_ws_layout(n, cin, c, ws, &s);
  const int cp = ce_cpad(c);
  k_ce_pad_w<<<(unsigned)ceil_div(cin * cp, 256), 256, 0, stream>>>(w, cin, c, cp, s.wp);
  OSB_LAUNCH_CHECK();
  const int64_t nblk = ce_row_blocks(n);
  if (labels_are_i64)
    k_ce_bwd_rows<int64_t><<<(unsigned)nblk, CE_THREADS, 0, stream>>>((const uint8_t *)x_split, n, cin, s.wp, c, cp, row_map,
                                                                       (const int64_t *)labels, (long long)ignore_index, lse, g,
                                                                       n_valid, s.d);
  else
    k_ce_bwd_rows<int32_t><<<(unsigned)nblk, CE_THREADS, 0, stream>>>((const uint8_t *)x_split, n, cin, s.wp, c, cp, row_map,
                                                                       (const int32_t *)labels, (long long)ignore_index, lse, g,
                                                                       n_valid, s.d);
  OSB_LAUNCH_CHECK();
  OSB_SMEM_ATTR_ONCE(k_ce_bwd_lines, ce_lines_smem(CE_MAX_C));
  const int64_t splits = ce_splits(n);
  k_ce_bwd_lines<<<dim3((unsigned)splits, (unsigned)(cin / 32)), CE_THREADS, ce_lines_smem(cp), stream>>>(
      (const uint8_t *)x_split, n, cin, s.wp, c, cp, s.d, (uint8_t *)dx_split, s.dwp);
  OSB_LAUNCH_CHECK();
  k_ce_dw_merge<<<(unsigned)ceil_div(cin * c, 256), 256, 0, stream>>>(s.dwp, splits, cin, c, cp, dw);
  OSB_LAUNCH_CHECK();
  return 0;
}

size_t osb_ce_head_eval_workspace_bytes(int64_t n_pts, int32_t cin, int32_t c) {
  if (n_pts < 0 || !ce_shape_ok(1, cin, c)) return 0;
  return ce_eval_ws_layout(n_pts, cin, c, nullptr, nullptr, nullptr);
}

int osb_ce_head_eval(const void *x_split, int64_t n_rows, int32_t cin, const float *w, int32_t c, const int32_t *row_map,
                     const int64_t *inds_reverse, int64_t n_pts, const void *labels, int32_t labels_are_i64,
                     int32_t ignore_index, int64_t *pred, float *loss, uint64_t *areas, int32_t *bad_labels, void *ws,
                     size_t ws_bytes, void *stream_) {
  const char *fn = "osb_ce_head_eval";
  OSB_CHECK(n_rows >= 1, "%s: rows (%lld) must be positive", fn, (long long)n_rows);
  OSB_CHECK(n_pts >= 0, "%s: points (%lld) must not be negative", fn, (long long)n_pts);
  OSB_CHECK(inds_reverse || n_pts == n_rows || n_pts == 0, "%s: without inds_reverse every row is one point (%lld points, %lld rows)", fn,
            (long long)n_pts, (long long)n_rows);
  OSB_CHECK(cin >= 32 && cin <= CE_MAX_CIN && cin % 32 == 0, "%s: input channels (%d) must be a multiple of 32 up to %d", fn, cin,
            CE_MAX_CIN);
  OSB_CHECK(c >= 1 && c <= CE_MAX_C, "%s: classes (%d) must be 1 to %d", fn, c, CE_MAX_C);
  OSB_CHECK(x_split && w && row_map && (labels || n_pts == 0), "%s: null rows, weights, row map or labels", fn);
  OSB_CHECK(loss && areas && bad_labels, "%s: null loss, areas or bad-label count", fn);
  OSB_CHECK(labels_are_i64 == 0 || labels_are_i64 == 1, "%s: labels_are_i64 must be 0 or 1", fn);
  OSB_CHECK(((uintptr_t)x_split & 15) == 0, "%s: rows must be 16-byte aligned", fn);
  const size_t need = ce_eval_ws_layout(n_pts, cin, c, nullptr, nullptr, nullptr);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 255) == 0,
            "%s: 256-byte aligned workspace of %zu bytes required (got %zu)", fn, need, ws_bytes);
  cudaStream_t stream = (cudaStream_t)stream_;
  CeWs s;
  int64_t *n_valid;
  ce_eval_ws_layout(n_pts, cin, c, ws, &s, &n_valid);
  const int cp = ce_cpad(c);
  const int64_t nblk = ce_row_blocks(n_pts);
  if (n_pts > 0) {
    k_ce_pad_w<<<(unsigned)ceil_div(cin * cp, 256), 256, 0, stream>>>(w, cin, c, cp, s.wp);
    OSB_LAUNCH_CHECK();
    if (labels_are_i64)
      k_ce_fwd_eval<int64_t><<<(unsigned)nblk, CE_THREADS, 0, stream>>>(
          (const uint8_t *)x_split, n_pts, cin, s.wp, c, cp, row_map, inds_reverse, (const int64_t *)labels, ignore_index, pred,
          s.part, (unsigned long long *)areas, bad_labels);
    else
      k_ce_fwd_eval<int32_t><<<(unsigned)nblk, CE_THREADS, 0, stream>>>(
          (const uint8_t *)x_split, n_pts, cin, s.wp, c, cp, row_map, inds_reverse, (const int32_t *)labels, ignore_index, pred,
          s.part, (unsigned long long *)areas, bad_labels);
    OSB_LAUNCH_CHECK();
  }
  k_ce_loss<<<1, CE_THREADS, 0, stream>>>(s.part, nblk, loss, n_valid);     // no point: 0 / 0 = NaN
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
