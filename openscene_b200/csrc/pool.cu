// Sparse pooling on CUDA cores (fp32): MinkowskiSumPooling / MinkowskiAvgPooling / MinkowskiMaxPooling over a kernel map,
// and MinkowskiGlobalSum/Avg/MaxPooling per batch index (models/resnet_base.py:54,68).
//
// Local pooling is output-stationary over the map a convolution with the same arguments uses (nbr[K][n_out]); the backward
// runs the same walk over the transposed map.  One thread owns one row and four channels (a float4 when the rows are 16-byte
// aligned, scalar loads otherwise) and walks the offsets in ascending k, so every output is written once, in a fixed order,
// without atomics: two runs give the same bits.
//   sum  s[o] = fp32 adds over the present offsets, ascending k, from +0.0
//   avg  s[o] / fp32(max(count_o, 1))
//   max  the largest present input; the first NaN in offset order wins, ties (+-0 included) go to the lowest k; an output
//        with no present input is 0.  The winning k is stored per (row, channel) in 16 bits (kNoWinner = none).
//
// Global pooling runs in two launches.  Rows are cut into chunks in .F order; a thread owns (chunk, channel) and walks the
// chunk's rows, keeping a running value for the current batch index and folding it into its private partial slot
// [chunk][batch][channel] whenever the index changes (batches may interleave).  A second launch merges the slots of each
// (batch, channel) in chunk order: fp64 for sum / avg, rounded to fp32 once; (value, row) for max.
#include "common.cuh"
#include <algorithm>

namespace osb {

enum { POOL_SUM = 0, POOL_AVG = 1, POOL_MAX = 2 };
constexpr uint16_t kNoWinner = 0xFFFF;
constexpr int POOL_THREADS = 256;
constexpr int64_t POOL_MAX_BLOCKS = 132 * 16;
constexpr int64_t GPOOL_CHUNK_ROWS = 256;                    // rows per chunk unless the workspace budget asks for more
constexpr int64_t GPOOL_WS_BUDGET = (int64_t)64 << 20;       // bytes of partial slots

// does v replace the current maximum `best`?  NaN is sticky, the first NaN wins, ties keep the earlier candidate
__device__ __forceinline__ bool max_takes(float best, float v) { return !(best != best) && ((v != v) || v > best); }

template <bool VEC>
__device__ __forceinline__ void load4(const float *__restrict__ p, int w, float (&v)[4]) {
  if (VEC) {
    const float4 q = __ldg(reinterpret_cast<const float4 *>(p));
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = j < w ? __ldg(p + j) : 0.f;
  }
}

template <bool VEC>
__device__ __forceinline__ void store4(float *__restrict__ p, int w, const float (&v)[4]) {
  if (VEC) {
    *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (j < w) p[j] = v[j];
  }
}

template <int MODE, bool VEC>
__global__ void __launch_bounds__(POOL_THREADS)
k_pool_fwd(const float *__restrict__ in, int c, const int32_t *__restrict__ nbr, int64_t n_out, int K, int tx_shift,
           float *__restrict__ out, int32_t *__restrict__ count, uint16_t *__restrict__ argk) {
  const int nch = (c + 3) >> 2;
  const int tx = threadIdx.x & ((1 << tx_shift) - 1), rpb = POOL_THREADS >> tx_shift;
  for (int64_t o = (int64_t)blockIdx.x * rpb + (threadIdx.x >> tx_shift); o < n_out; o += (int64_t)gridDim.x * rpb)
  for (int ch = tx; ch < nch; ch += 1 << tx_shift) {
    const int c0 = ch * 4;
    const int w = min(4, c - c0);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    int win[4] = {kNoWinner, kNoWinner, kNoWinner, kNoWinner};
    int n = 0;
    for (int k = 0; k < K; ++k) {
      const int32_t i = __ldg(nbr + (int64_t)k * n_out + o);
      if (i < 0) continue;
      ++n;
      float v[4];
      load4<VEC>(in + (int64_t)i * c + c0, w, v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (MODE == POOL_MAX) {
          if (win[j] == kNoWinner || max_takes(acc[j], v[j])) { acc[j] = v[j]; win[j] = k; }
        } else {
          acc[j] = __fadd_rn(acc[j], v[j]);
        }
      }
    }
    if (MODE == POOL_AVG) {
      const float d = (float)max(n, 1);
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[j] = __fdiv_rn(acc[j], d);
      if (c0 == 0) count[o] = n;
    }
    store4<VEC>(out + o * c + c0, w, acc);
    if (MODE == POOL_MAX) {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (j < w) argk[o * c + c0 + j] = (uint16_t)win[j];
    }
  }
}

// gin[i] = sum over ascending k of the term of the output o = nbr_t[k][i]: g[o] (sum), fp32(g[o] / count_o) (avg), g[o] where
// the stored winner of (o, channel) is k (max)
template <int MODE, bool VEC>
__global__ void __launch_bounds__(POOL_THREADS)
k_pool_bwd(const float *__restrict__ gout, int c, const int32_t *__restrict__ nbr_t, int64_t n_in, int K, int tx_shift,
           const int32_t *__restrict__ count, const uint16_t *__restrict__ argk, float *__restrict__ gin) {
  const int nch = (c + 3) >> 2;
  const int tx = threadIdx.x & ((1 << tx_shift) - 1), rpb = POOL_THREADS >> tx_shift;
  for (int64_t i = (int64_t)blockIdx.x * rpb + (threadIdx.x >> tx_shift); i < n_in; i += (int64_t)gridDim.x * rpb)
  for (int ch = tx; ch < nch; ch += 1 << tx_shift) {
    const int c0 = ch * 4;
    const int w = min(4, c - c0);
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int k = 0; k < K; ++k) {
      const int32_t o = __ldg(nbr_t + (int64_t)k * n_in + i);
      if (o < 0) continue;
      float g[4];
      load4<VEC>(gout + (int64_t)o * c + c0, w, g);
      if (MODE == POOL_AVG) {
        const float d = (float)max(__ldg(count + o), 1);
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = __fadd_rn(acc[j], __fdiv_rn(g[j], d));
      } else if (MODE == POOL_MAX) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < w && __ldg(argk + (int64_t)o * c + c0 + j) == (uint16_t)k) acc[j] = __fadd_rn(acc[j], g[j]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[j] = __fadd_rn(acc[j], g[j]);
      }
    }
    store4<VEC>(gin + i * c + c0, w, acc);
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// global pooling
struct MaxSlot {
  float v;
  int32_t row;  // -1: no row yet
};

struct GPoolPlan {
  int64_t chunk_rows, n_chunks;
  size_t slot_bytes, count_bytes;
};

static GPoolPlan gpool_plan(int64_t n, int c, int n_batch) {
  GPoolPlan p{0, 0, 0, 0};
  if (n < 1 || c < 1 || n_batch < 1) return p;
  const int64_t per_chunk = (int64_t)n_batch * c * 8;
  const int64_t max_chunks = std::max<int64_t>(1, GPOOL_WS_BUDGET / per_chunk);
  p.chunk_rows = std::max(GPOOL_CHUNK_ROWS, ceil_div(n, max_chunks));
  p.n_chunks = ceil_div(n, p.chunk_rows);
  p.slot_bytes = (size_t)(ceil_div(p.n_chunks * per_chunk, 256) * 256);
  p.count_bytes = (size_t)p.n_chunks * n_batch * sizeof(int32_t);
  return p;
}

template <int MODE>
__global__ void __launch_bounds__(POOL_THREADS)
k_gpool_partial(const float *__restrict__ in, const int32_t *__restrict__ batch, int64_t n, int c, int n_batch,
                int64_t chunk_rows, int64_t n_chunks, void *__restrict__ slots_, int32_t *__restrict__ counts) {
  const int64_t total = n_chunks * c;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = e / c;
    const int cc = (int)(e - j * c);
    const int64_t r0 = j * chunk_rows, r1 = min(r0 + chunk_rows, n);
    int cur = -1;
    double run = 0.0;
    int32_t cnt = 0;
    float best = 0.f;
    int32_t best_row = -1;
    auto flush = [&]() {
      if (cur < 0) return;
      const int64_t s = (j * n_batch + cur) * c + cc;
      if (MODE == POOL_MAX) {
        MaxSlot *slots = reinterpret_cast<MaxSlot *>(slots_);
        const MaxSlot m = slots[s];
        if (m.row < 0 || max_takes(m.v, best)) slots[s] = MaxSlot{best, best_row};
      } else {
        double *slots = reinterpret_cast<double *>(slots_);
        slots[s] = __dadd_rn(slots[s], run);
        if (MODE == POOL_AVG && cc == 0) counts[j * n_batch + cur] += cnt;
      }
    };
    for (int64_t r = r0; r < r1; ++r) {
      const int b = __ldg(batch + r);
      const float v = __ldg(in + r * c + cc);
      if (b != cur) {
        flush();
        cur = b, run = 0.0, cnt = 0, best_row = -1;
      }
      if (MODE == POOL_MAX) {
        if (best_row < 0 || max_takes(best, v)) best = v, best_row = (int32_t)r;
      } else {
        run = __dadd_rn(run, (double)v);
        ++cnt;
      }
    }
    flush();
  }
}

template <int MODE>
__global__ void __launch_bounds__(POOL_THREADS)
k_gpool_merge(int c, int n_batch, int64_t n_chunks, const void *__restrict__ slots_, const int32_t *__restrict__ counts,
              float *__restrict__ out, int32_t *__restrict__ count_out, int32_t *__restrict__ argrow) {
  const int64_t total = (int64_t)n_batch * c;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(e / c);
    const int cc = (int)(e - (int64_t)b * c);
    if (MODE == POOL_MAX) {
      const MaxSlot *slots = reinterpret_cast<const MaxSlot *>(slots_);
      float best = 0.f;
      int32_t row = -1;
      for (int64_t j = 0; j < n_chunks; ++j) {
        const MaxSlot m = slots[(j * n_batch + b) * c + cc];
        if (m.row >= 0 && (row < 0 || max_takes(best, m.v))) best = m.v, row = m.row;
      }
      out[e] = row < 0 ? -INFINITY : best;
      argrow[e] = row;
    } else {
      const double *slots = reinterpret_cast<const double *>(slots_);
      double acc = 0.0;
      int64_t cnt = 0;
#pragma unroll 4
      for (int64_t j = 0; j < n_chunks; ++j) {
        acc = __dadd_rn(acc, slots[(j * n_batch + b) * c + cc]);
        if (MODE == POOL_AVG) cnt += __ldg(counts + j * n_batch + b);
      }
      if (MODE == POOL_AVG) {
        out[e] = (float)__ddiv_rn(acc, (double)cnt);            // an empty batch: 0 / 0 = NaN
        if (cc == 0) count_out[b] = (int32_t)cnt;
      } else {
        out[e] = (float)acc;
      }
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(POOL_THREADS)
k_gpool_bwd(const float *__restrict__ gout, const int32_t *__restrict__ batch, int64_t n, int c, const int32_t *__restrict__ count,
            const int32_t *__restrict__ argrow, float *__restrict__ gin) {
  const int64_t total = n * c;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / c;
    const int cc = (int)(e - r * c);
    const int b = __ldg(batch + r);
    const int64_t s = (int64_t)b * c + cc;
    const float g = __ldg(gout + s);
    float v;
    if (MODE == POOL_SUM) v = g;
    else if (MODE == POOL_AVG) v = __fdiv_rn(g, (float)__ldg(count + b));
    else v = __ldg(argrow + s) == (int32_t)r ? g : 0.f;
    gin[e] = v;
  }
}

static unsigned grid_blocks(int64_t total) { return (unsigned)std::max<int64_t>(1, std::min(ceil_div(total, POOL_THREADS), POOL_MAX_BLOCKS)); }

// local pooling launch plan: a block is 2^(8 - shift) rows x 2^shift lanes of four channels, lanes = the channel groups rounded
// up to a power of two (at most 64; wider rows loop over their groups)
static int pool_tx_shift(int c) {
  const int nch = (c + 3) / 4;
  int sh = 0;
  while ((1 << sh) < nch && sh < 6) ++sh;
  return sh;
}
static unsigned pool_blocks(int64_t rows, int sh) {
  return (unsigned)std::max<int64_t>(1, std::min(ceil_div(rows, POOL_THREADS >> sh), POOL_MAX_BLOCKS));
}

static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int MODE>
static int launch_pool_fwd(const float *in, int c, const int32_t *nbr, int64_t n_out, int K, float *out, int32_t *count,
                           uint16_t *argk, cudaStream_t stream) {
  const int sh = pool_tx_shift(c);
  const unsigned grid = pool_blocks(n_out, sh);
  if ((c & 3) == 0 && aligned16(in) && aligned16(out))
    k_pool_fwd<MODE, true><<<grid, POOL_THREADS, 0, stream>>>(in, c, nbr, n_out, K, sh, out, count, argk);
  else
    k_pool_fwd<MODE, false><<<grid, POOL_THREADS, 0, stream>>>(in, c, nbr, n_out, K, sh, out, count, argk);
  OSB_LAUNCH_CHECK();
  return 0;
}

template <int MODE>
static int launch_pool_bwd(const float *gout, int c, const int32_t *nbr_t, int64_t n_in, int K, const int32_t *count,
                           const uint16_t *argk, float *gin, cudaStream_t stream) {
  const int sh = pool_tx_shift(c);
  const unsigned grid = pool_blocks(n_in, sh);
  if ((c & 3) == 0 && aligned16(gout) && aligned16(gin))
    k_pool_bwd<MODE, true><<<grid, POOL_THREADS, 0, stream>>>(gout, c, nbr_t, n_in, K, sh, count, argk, gin);
  else
    k_pool_bwd<MODE, false><<<grid, POOL_THREADS, 0, stream>>>(gout, c, nbr_t, n_in, K, sh, count, argk, gin);
  OSB_LAUNCH_CHECK();
  return 0;
}

template <int MODE>
static int launch_gpool_fwd(const float *in, const int32_t *batch, int64_t n, int c, int n_batch, float *out, int32_t *count,
                            int32_t *argrow, void *ws, const GPoolPlan &p, cudaStream_t stream) {
  int32_t *counts = reinterpret_cast<int32_t *>(static_cast<char *>(ws) + p.slot_bytes);
  OSB_CUDA(cudaMemsetAsync(ws, MODE == POOL_MAX ? 0xFF : 0, p.slot_bytes + p.count_bytes, stream));
  k_gpool_partial<MODE><<<grid_blocks(p.n_chunks * c), POOL_THREADS, 0, stream>>>(in, batch, n, c, n_batch, p.chunk_rows,
                                                                                   p.n_chunks, ws, counts);
  OSB_LAUNCH_CHECK();
  k_gpool_merge<MODE><<<grid_blocks((int64_t)n_batch * c), POOL_THREADS, 0, stream>>>(c, n_batch, p.n_chunks, ws, counts, out,
                                                                                       count, argrow);
  OSB_LAUNCH_CHECK();
  return 0;
}

template <int MODE>
static int launch_gpool_bwd(const float *gout, const int32_t *batch, int64_t n, int c, const int32_t *count, const int32_t *argrow,
                            float *gin, cudaStream_t stream) {
  k_gpool_bwd<MODE><<<grid_blocks(n * c), POOL_THREADS, 0, stream>>>(gout, batch, n, c, count, argrow, gin);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // namespace osb

using namespace osb;

extern "C" {

int osb_pool_fwd(const float *in, int32_t c, const int32_t *nbr, int64_t n_out, int32_t K, int32_t mode, float *out,
                 int32_t *count, uint16_t *argk, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(mode >= POOL_SUM && mode <= POOL_MAX, "osb_pool_fwd: bad mode %d (0 sum, 1 avg, 2 max)", mode);
  OSB_CHECK(n_out >= 1 && c >= 1, "osb_pool_fwd: bad shape (n_out %lld, c %d)", (long long)n_out, c);
  OSB_CHECK(K >= 1 && K <= 65535, "osb_pool_fwd: K %d outside 1..65535", K);
  OSB_CHECK(in && nbr && out, "osb_pool_fwd: NULL buffer (in %p, nbr %p, out %p)", (const void *)in, (const void *)nbr, (void *)out);
  OSB_CHECK(mode != POOL_AVG || count, "osb_pool_fwd: average pooling needs the count buffer");
  OSB_CHECK(mode != POOL_MAX || argk, "osb_pool_fwd: max pooling needs the winner buffer");
  switch (mode) {
    case POOL_SUM: return launch_pool_fwd<POOL_SUM>(in, c, nbr, n_out, K, out, count, argk, stream);
    case POOL_AVG: return launch_pool_fwd<POOL_AVG>(in, c, nbr, n_out, K, out, count, argk, stream);
    default: return launch_pool_fwd<POOL_MAX>(in, c, nbr, n_out, K, out, count, argk, stream);
  }
}

int osb_pool_bwd(const float *gout, int32_t c, const int32_t *nbr_t, int64_t n_in, int32_t K, int32_t mode, const int32_t *count,
                 const uint16_t *argk, float *gin, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(mode >= POOL_SUM && mode <= POOL_MAX, "osb_pool_bwd: bad mode %d (0 sum, 1 avg, 2 max)", mode);
  OSB_CHECK(n_in >= 1 && c >= 1, "osb_pool_bwd: bad shape (n_in %lld, c %d)", (long long)n_in, c);
  OSB_CHECK(K >= 1 && K <= 65535, "osb_pool_bwd: K %d outside 1..65535", K);
  OSB_CHECK(gout && nbr_t && gin, "osb_pool_bwd: NULL buffer (gout %p, nbr_t %p, gin %p)", (const void *)gout, (const void *)nbr_t,
            (void *)gin);
  OSB_CHECK(mode != POOL_AVG || count, "osb_pool_bwd: average pooling needs the count buffer");
  OSB_CHECK(mode != POOL_MAX || argk, "osb_pool_bwd: max pooling needs the winner buffer");
  switch (mode) {
    case POOL_SUM: return launch_pool_bwd<POOL_SUM>(gout, c, nbr_t, n_in, K, count, argk, gin, stream);
    case POOL_AVG: return launch_pool_bwd<POOL_AVG>(gout, c, nbr_t, n_in, K, count, argk, gin, stream);
    default: return launch_pool_bwd<POOL_MAX>(gout, c, nbr_t, n_in, K, count, argk, gin, stream);
  }
}

size_t osb_global_pool_workspace_bytes(int64_t n, int32_t c, int32_t n_batch) {
  const GPoolPlan p = gpool_plan(n, c, n_batch);
  return p.slot_bytes + p.count_bytes;
}

int osb_global_pool_fwd(const float *in, const int32_t *batch, int64_t n, int32_t c, int32_t n_batch, int32_t mode, float *out,
                        int32_t *count, int32_t *argrow, void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(mode >= POOL_SUM && mode <= POOL_MAX, "osb_global_pool_fwd: bad mode %d (0 sum, 1 avg, 2 max)", mode);
  OSB_CHECK(n >= 1 && c >= 1 && n_batch >= 1, "osb_global_pool_fwd: bad shape (n %lld, c %d, n_batch %d)", (long long)n, c, n_batch);
  OSB_CHECK(in && batch && out, "osb_global_pool_fwd: NULL buffer (in %p, batch %p, out %p)", (const void *)in, (const void *)batch,
            (void *)out);
  OSB_CHECK(mode != POOL_AVG || count, "osb_global_pool_fwd: average pooling needs the count buffer");
  OSB_CHECK(mode != POOL_MAX || argrow, "osb_global_pool_fwd: max pooling needs the winner buffer");
  const GPoolPlan p = gpool_plan(n, c, n_batch);
  OSB_CHECK(ws && aligned16(ws), "osb_global_pool_fwd: workspace %p is NULL or not 16-byte aligned", ws);
  OSB_CHECK(ws_bytes >= p.slot_bytes + p.count_bytes, "osb_global_pool_fwd: workspace of %zu bytes, %zu needed", ws_bytes,
            p.slot_bytes + p.count_bytes);
  switch (mode) {
    case POOL_SUM: return launch_gpool_fwd<POOL_SUM>(in, batch, n, c, n_batch, out, count, argrow, ws, p, stream);
    case POOL_AVG: return launch_gpool_fwd<POOL_AVG>(in, batch, n, c, n_batch, out, count, argrow, ws, p, stream);
    default: return launch_gpool_fwd<POOL_MAX>(in, batch, n, c, n_batch, out, count, argrow, ws, p, stream);
  }
}

int osb_global_pool_bwd(const float *gout, const int32_t *batch, int64_t n, int32_t c, int32_t mode, const int32_t *count,
                        const int32_t *argrow, float *gin, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(mode >= POOL_SUM && mode <= POOL_MAX, "osb_global_pool_bwd: bad mode %d (0 sum, 1 avg, 2 max)", mode);
  OSB_CHECK(n >= 1 && c >= 1, "osb_global_pool_bwd: bad shape (n %lld, c %d)", (long long)n, c);
  OSB_CHECK(gout && batch && gin, "osb_global_pool_bwd: NULL buffer (gout %p, batch %p, gin %p)", (const void *)gout,
            (const void *)batch, (void *)gin);
  OSB_CHECK(mode != POOL_AVG || count, "osb_global_pool_bwd: average pooling needs the count buffer");
  OSB_CHECK(mode != POOL_MAX || argrow, "osb_global_pool_bwd: max pooling needs the winner buffer");
  switch (mode) {
    case POOL_SUM: return launch_gpool_bwd<POOL_SUM>(gout, batch, n, c, count, argrow, gin, stream);
    case POOL_AVG: return launch_gpool_bwd<POOL_AVG>(gout, batch, n, c, count, argrow, gin, stream);
    default: return launch_gpool_bwd<POOL_MAX>(gout, batch, n, c, count, argrow, gin, stream);
  }
}

}  // extern "C"
