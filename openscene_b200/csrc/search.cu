// Scene search (DESIGN.md, "Scene search contract"): a few query embeddings against every row of a database of scenes.
//
//   s[r, q] = fp16( sum_c A[r, c] * Q[q, c] )      the bits osb_match_scores writes for fp16 rows, normalize = 0
//
// Per query the k best rows of the whole index, and per scene and query the best score, its row and the number of rows
// scoring at or above a threshold.  The [N, nq] scores never reach memory.
//
// k_search is a persistent loop over 128-row tiles (one CTA per SM).  Per tile, the A producers of the tensor-core match
// (match_tc.cuh) load the rows and write the K-major operand, warp 16 streams the query chunks with TMA, and warps 0-7 run
// the match kernel's wgmma pass and round to fp16.  The tile's fp16 scores then go to shared memory (over the A tile, which
// the product no longer needs), and four threads per query scan a column each over 32 rows:
//   - each run of one scene folds into (max order key, count); a tile inside one scene costs one 64-bit atomicMax and one
//     integer add per query, a tile that crosses scenes one per run and quarter;
//   - keys above the k-th key of the CTA's running list (global, L2-resident) are inserted into it, one lane of the
//     quad at a time.
// While the tile is multiplied and scanned, the producers have already asked L2 for the next tile's rows.
// k_search_finish merges the per-CTA lists into the k best keys per query and decodes keys into (score, scene, row), and
// decodes the per-scene keys and counts.
//
// Order key (search_key): bits 48-63 the score's order (-0 as +0), bits 16-47 ~row (the lower global row wins a tie), bits
// 0-15 the score's fp16 bits; NaN has key 0, below every other key, so it never ranks, is never a maximum and is never
// counted.  Keys are distinct, so the top-k is a function of the scores alone, and atomicMax / integer adds make the
// per-scene results independent of the order in which CTAs arrive.
#include "match_tc.cuh"
#include "sortscan.cuh"
#include <algorithm>

namespace osb {

constexpr int SR_LD = MT_NW + 8;           // fp16 score tile: row stride in halves
constexpr int SR_MAX_GRID = 132;           // CTAs: one per SM of an H100 SXM at most (the workspace is sized for it)

struct SearchParams {
  MatchTcParams a;                         // the operand: fp16 rows, no gather, no normalisation
  const int32_t *row_scene;                // [n] scene of every row
  int64_t n, n_tiles;
  int nq, k;
  const float *thr;                        // [nq] or NULL (nothing counted)
  uint64_t *lists;                         // [gridDim.x][nq][k] running top-k keys, descending
  unsigned long long *scene_key;           // [S][nq] max key, 0 = none
  unsigned long long *scene_cnt;           // [S][nq]
  // hit emission (k_search<NP, true> only)
  int64_t n_scenes;
  unsigned long long *cursor;              // [nq][S] next free slot of each (query, scene) segment of the hit list
  const unsigned long long *seg_end;       // [nq][S] end of each segment
  uint64_t *hit_key;                       // [n_hits] (query << 32) | global row, in arrival order
  __half *hit_score;                       // [n_hits]
  int *status;                             // OSB_REGIONS_ST_COUNT when a segment's hits do not match its count
  const int8_t *row_exp;                   // [n] FP8 storage (k_search<NP, HITS, true>): a.feat holds e4m3 codes [n, C]
};

__device__ __forceinline__ void scene_flush(const SearchParams &sp, int s, int q, uint64_t key, uint32_t cnt) {
  if (s < 0) return;
  const size_t i = (size_t)s * sp.nq + q;
  if (key) atomicMax(sp.scene_key + i, (unsigned long long)key);
  if (cnt) atomicAdd(sp.scene_cnt + i, (unsigned long long)cnt);
}

// the hits of one scene run of a thread's 32 rows (bit j = row 32 qu + j) into their (query, scene) segment
__device__ __forceinline__ void hit_flush(const SearchParams &sp, const __half *sS, int64_t row0, int qu, int q, int s,
                                          uint32_t hm) {
  if (hm == 0) return;
  const size_t seg = (size_t)q * sp.n_scenes + s;
  const uint32_t n = __popc(hm);
  unsigned long long pos = atomicAdd(sp.cursor + seg, (unsigned long long)n);
  if (pos + n > sp.seg_end[seg]) { atomicOr(sp.status, OSB_REGIONS_ST_COUNT); return; }
  while (hm) {
    const int j = __ffs(hm) - 1;
    hm &= hm - 1;
    const int r = 32 * qu + j;
    sp.hit_key[pos] = ((uint64_t)q << 32) | (uint64_t)(row0 + r);
    sp.hit_score[pos] = sS[r * SR_LD + q];
    ++pos;
  }
}

__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// HITS = false: the search epilogue below.  HITS = true: the same loads, query stream and product; the epilogue writes
// every (row, query) with float(s) >= thr[q] into the hit list instead (osb_search_hits).  F8 = true: the rows are e4m3
// codes with per-row exponents (osb_search_f8, osb_search_hits_f8); mt_fill_a8 writes the tile mt_fill_a writes for their
// dequantized fp16 rows, and everything after the tile is the same.
template <int NP, bool HITS = false, bool F8 = false>
__global__ void __launch_bounds__(MT_THREADS, 1) k_search(const __grid_constant__ CUtensorMap tmQ, const SearchParams sp) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int C = 64 * NP;
  constexpr int A_BYTES = NP * MT_M * 128, B_BYTES = MT_NW * 128;
  uint8_t *sA = smem, *sB = smem + A_BYTES;
  uint64_t *bars = reinterpret_cast<uint64_t *>(sB + MT_BSTAGES * B_BYTES);   // b_full[2], b_empty[2]
  int32_t *s_scene = reinterpret_cast<int32_t *>(sB + MT_BSTAGES * B_BYTES + 128);
  __half *sS = reinterpret_cast<__half *>(sA);                                 // [128][SR_LD] once the product is done

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t b_full = smem_u32(bars), b_empty = smem_u32(bars + 2);
  uint64_t *lists = sp.lists + (size_t)blockIdx.x * sp.nq * sp.k;
  if (tid == 0) {
    for (int s = 0; s < MT_BSTAGES; ++s) { mbar_init(b_full + 8 * s, 1); mbar_init(b_empty + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid == MT_PW * 32) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmQ) : "memory");
  if constexpr (!HITS)
    for (int i = tid; i < sp.nq * sp.k; i += MT_THREADS) lists[i] = 0;   // empty lists: key 0 is below every valid key
  __syncthreads();

  if (warp == MT_PW) {
    // ============================ TMA producer: the query chunks of every tile ============================
    int s = 0; uint32_t phase = 0;
    for (int64_t t = blockIdx.x; t < sp.n_tiles; t += gridDim.x)
      for (int c = 0; c < NP; ++c) mt_text_stage(tmQ, sB, b_full, b_empty, c, 0, s, phase);
    return;
  }

  // warps 0-15 from here on; they synchronise on named barrier 1
  int s = 0; uint32_t phase = 0;
  for (int64_t t = blockIdx.x; t < sp.n_tiles; t += gridDim.x) {
    const int64_t row0 = t * MT_M;
    const int nrows = (int)std::min<int64_t>(MT_M, sp.n - row0);
    {   // the next tile's rows into L2 while this one is loaded, multiplied and scanned
      const int64_t nt = t + gridDim.x;
      constexpr int ROW_BYTES = F8 ? C : 2 * C;
      if (nt < sp.n_tiles) {
        const char *base = reinterpret_cast<const char *>(sp.a.feat) + nt * MT_M * (int64_t)ROW_BYTES;
        const int64_t bytes = std::min<int64_t>(MT_M, sp.n - nt * MT_M) * ROW_BYTES;
        for (int64_t o = (int64_t)tid * 128; o < bytes; o += MT_PW * 32 * 128)
          asm volatile("prefetch.global.L2 [%0];" ::"l"(base + o));
        if (F8 && tid == MT_PW * 32 - 1) asm volatile("prefetch.global.L2 [%0];" ::"l"(sp.row_exp + nt * MT_M));
      }
    }
    if (tid < MT_M) s_scene[tid] = tid < nrows ? __ldg(sp.row_scene + row0 + tid) : -1;
    if constexpr (F8)
      mt_fill_a8<NP>(reinterpret_cast<const uint8_t *>(sp.a.feat), sp.row_exp, sp.n, sA, row0, warp, lane);
    else
      mt_fill_a<NP>(sp.a, sA, row0, warp, lane);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");           // generic-proxy writes -> wgmma reads
    bar_sync(1, MT_PW * 32);

    if (warp < 8) {
      // ============ wgmma: warpgroup g multiplies rows [64g, 64g + 64) by the query block; fp16 scores to sS ============
      const int g = warp >> 2;
      float acc[MT_NW / 2];
#pragma unroll
      for (int i = 0; i < MT_NW / 2; ++i) acc[i] = 0.f;
      mt_mma_pass<NP>(acc, sA, sB, g, tid, b_full, b_empty, s, phase);
      bar_sync(2, 256);                                                    // both warpgroups are done reading sA
      const int r_lo = 64 * g + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < MT_NW / 8; ++i)
          *reinterpret_cast<__half2 *>(sS + (r_lo + 8 * h) * SR_LD + 8 * i + cq) =
              __floats2half2_rn(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
    }
    bar_sync(1, MT_PW * 32);

    if constexpr (HITS) {
      // ============ hit emission: query q = tid / 4, rows 32 qu .. 32 qu + 31, one segment cursor update per scene run ============
      const int q = tid >> 2, qu = tid & 3;
      if (tid < 4 * MT_NW && q < sp.nq) {
        const float th = __ldg(sp.thr + q);
        int cur = -1;
        uint32_t hm = 0;
        for (int j = 0; j < 32; ++j) {
          const int r = 32 * qu + j;
          if (r >= nrows) break;
          const int sc = s_scene[r];
          if (sc != cur) { if (cur >= 0) hit_flush(sp, sS, row0, qu, q, cur, hm); cur = sc; hm = 0; }
          if (__half2float(sS[r * SR_LD + q]) >= th) hm |= 1u << j;
        }
        if (cur >= 0) hit_flush(sp, sS, row0, qu, q, cur, hm);
      }
    } else if (tid < 4 * MT_NW) {
      // ============ column scan: query q = tid / 4, rows 32 qu .. 32 qu + 31 (qu = tid % 4) ============
      const int q = tid >> 2, qu = tid & 3;
      const bool act = q < sp.nq;
      const int first = s_scene[0];
      const bool one = first == s_scene[nrows - 1];                        // scene ids ascend with the row
      const float th = (act && sp.thr) ? __ldg(sp.thr + q) : __int_as_float(0x7fc00000);
      uint64_t *L = lists + (size_t)(act ? q : 0) * sp.k;
      const uint64_t kth = act ? L[sp.k - 1] : ~0ull;
      uint64_t mk = 0;
      uint32_t cnt = 0, cand = 0;
      int cur = -1;
      if (act) {
        for (int j = 0; j < 32; ++j) {
          const int r = 32 * qu + j;
          if (r >= nrows) break;
          const int sc = s_scene[r];
          const __half h = sS[r * SR_LD + q];
          const uint64_t key = search_key(h, row0 + r);
          if (sc != cur) { scene_flush(sp, cur, q, mk, cnt); cur = sc; mk = 0; cnt = 0; }
          mk = std::max(mk, key);
          cnt += __half2float(h) >= th ? 1u : 0u;
          if (key > kth) cand |= 1u << j;
        }
      }
      if (one) {   // one scene: merge the quad, one update per query
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          mk = std::max(mk, (uint64_t)__shfl_xor_sync(0xffffffffu, (unsigned long long)mk, o));
          cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        }
        if (qu == 0 && act) scene_flush(sp, first, q, mk, cnt);
      } else if (act) {
        scene_flush(sp, cur, q, mk, cnt);
      }
      if (__any_sync(0xffffffffu, cand != 0)) {   // the candidates, one lane of each quad at a time
#pragma unroll 1
        for (int w = 0; w < 4; ++w) {
          if (qu == w) {
            while (cand) {
              const int j = __ffs(cand) - 1;
              cand &= cand - 1;
              const int r = 32 * qu + j;
              topk_insert(L, sp.k, search_key(sS[r * SR_LD + q], row0 + r));
            }
          }
          __syncwarp();
        }
      }
    }
    bar_sync(1, MT_PW * 32);                                               // sS is read: the next tile may overwrite it
  }
}

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = std::max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// blocks 0 .. nq-1: the k best keys of query q over all CTA lists, decoded; the other blocks: the per-scene results
__global__ void __launch_bounds__(256)
k_search_finish(const uint64_t *__restrict__ lists, int n_lists, int nq, int k, const int32_t *__restrict__ row_scene,
                const int64_t *__restrict__ off, __half *top_score, int64_t *top_scene, int64_t *top_row,
                const unsigned long long *__restrict__ scene_key, const unsigned long long *__restrict__ scene_cnt,
                int64_t n_scenes, __half *scene_max, int64_t *scene_argmax, int64_t *scene_count) {
  const int tid = threadIdx.x;
  if ((int)blockIdx.x < nq) {
    extern __shared__ uint64_t s_keys[];
    __shared__ unsigned long long s_red[8];
    const int q = blockIdx.x, n = n_lists * k;
    for (int i = tid; i < n; i += 256) s_keys[i] = lists[((size_t)(i / k) * nq + q) * k + i % k];
    __syncthreads();
    uint64_t last = ~0ull;
    for (int j = 0; j < k; ++j) {   // round j: the largest key below the previous one (keys are distinct)
      unsigned long long m = 0;
      for (int i = tid; i < n; i += 256) {
        const uint64_t v = s_keys[i];
        if (v < last && v > m) m = v;
      }
      m = warp_max_u64(m);
      if ((tid & 31) == 0) s_red[tid >> 5] = m;
      __syncthreads();
      m = s_red[0];
      for (int w = 1; w < 8; ++w) m = std::max(m, s_red[w]);
      __syncthreads();
      last = m;
      if (tid == 0) {
        const size_t o = (size_t)q * k + j;
        if (m == 0) {   // fewer than k rows with a score
          top_score[o] = __ushort_as_half((unsigned short)0xfc00u);
          top_scene[o] = -1;
          top_row[o] = -1;
        } else {
          const int64_t grow = (int64_t)(~(uint32_t)(m >> 16));
          const int sc = row_scene[grow];
          top_score[o] = __ushort_as_half((unsigned short)(m & 0xffffu));
          top_scene[o] = sc;
          top_row[o] = grow - off[sc];
        }
      }
    }
    return;
  }
  const int64_t total = n_scenes * nq, stride = (int64_t)(gridDim.x - nq) * 256;
  for (int64_t i = (int64_t)(blockIdx.x - nq) * 256 + tid; i < total; i += stride) {
    const uint64_t key = scene_key[i];
    if (key == 0) {
      scene_max[i] = __ushort_as_half((unsigned short)0xfc00u);
      scene_argmax[i] = -1;
    } else {
      scene_max[i] = __ushort_as_half((unsigned short)(key & 0xffffu));
      scene_argmax[i] = (int64_t)(~(uint32_t)(key >> 16)) - off[i / nq];
    }
    if (scene_count) scene_count[i] = (int64_t)scene_cnt[i];
  }
}

// segments of the hit list in (query, scene) order: base = exclusive scan of scene_count[s][q] over (q, s); one block
__global__ void __launch_bounds__(1024)
k_hit_segments(const int64_t *__restrict__ scene_count, int64_t n_scenes, int nq, int64_t n_hits,
               unsigned long long *cursor, unsigned long long *seg_end, int *status) {
  __shared__ unsigned long long s_part[1024];
  const int64_t m = n_scenes * nq, per = (m + 1023) / 1024;
  const int64_t a = std::min<int64_t>(m, per * threadIdx.x), b = std::min<int64_t>(m, a + per);
  unsigned long long t = 0;
  for (int64_t i = a; i < b; ++i) t += (unsigned long long)scene_count[(i % n_scenes) * nq + i / n_scenes];
  s_part[threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int i = 0; i < 1024; ++i) { const unsigned long long v = s_part[i]; s_part[i] = run; run += v; }
    if (run != (unsigned long long)n_hits) atomicOr(status, OSB_REGIONS_ST_COUNT);
  }
  __syncthreads();
  unsigned long long run = s_part[threadIdx.x];
  for (int64_t i = a; i < b; ++i) {
    cursor[i] = run;
    run += (unsigned long long)scene_count[(i % n_scenes) * nq + i / n_scenes];
    seg_end[i] = std::min<unsigned long long>(run, (unsigned long long)n_hits);
  }
}

// the segments of a hit list whose counts [S][nq] are known (label.cu's class hits), as osb_search_hits lays them out
int hit_segments_run(const int64_t *scene_count, int64_t n_scenes, int nq, int64_t n_hits, unsigned long long *cursor,
                     unsigned long long *seg_end, int *status, cudaStream_t stream) {
  k_hit_segments<<<1, 1024, 0, stream>>>(scene_count, n_scenes, nq, n_hits, cursor, seg_end, status);
  OSB_LAUNCH_CHECK();
  return 0;
}

// every segment received exactly its count; the scores follow the sorted keys (payload = arrival slot)
__global__ void k_hit_finish(const unsigned long long *__restrict__ cursor, const unsigned long long *__restrict__ seg_end,
                             int64_t n_seg, const int32_t *__restrict__ slot, const __half *__restrict__ score_in,
                             int64_t n_hits, __half *score_out, int *status) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_seg; i += stride)
    if (cursor[i] != seg_end[i]) atomicOr(status, OSB_REGIONS_ST_COUNT);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_hits; i += stride) score_out[i] = score_in[slot[i]];
}

// FP8 index rows (DESIGN.md, "FP8 index contract"): one warp per row, 8 elements per lane and unit.  h = the row as fp16 (fp32
// rows are rounded first), amax = max |h| by a warp reduction, e the smallest integer with amax <= 448 * 2^e clamped to
// [-15, 7], codes = e4m3_rn(clamp(h * 2^-e, -448, 448)) by the hardware conversion; a row with a NaN or inf element gets NaN
// codes (0x7f) and e = 0.  h * 2^-e is exact in fp32, so the conversion is the only rounding.
template <int NP>
__global__ void __launch_bounds__(256) k_index_quantize_f8(const void *__restrict__ rows, int rows_are_f16, int64_t n,
                                                           uint8_t *__restrict__ codes, int8_t *__restrict__ row_exp) {
  constexpr int C = 64 * NP, U = NP / 4;
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * 8;
  for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n; r += warps) {
    float v[U][8];
    if (rows_are_f16) {
      const uint4 *src = reinterpret_cast<const uint4 *>(rows) + r * (C / 8);
#pragma unroll
      for (int i = 0; i < U; ++i) {
        const uint4 x = __ldg(src + lane + 32 * i);
        const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2 *>(&w[p]));
          v[i][2 * p] = f.x; v[i][2 * p + 1] = f.y;
        }
      }
    } else {
      const float4 *src = reinterpret_cast<const float4 *>(rows) + r * (C / 4);
#pragma unroll
      for (int i = 0; i < U; ++i) {
        const float4 a = __ldg(src + 2 * (lane + 32 * i)), b = __ldg(src + 2 * (lane + 32 * i) + 1);
        const float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) v[i][j] = __half2float(__float2half_rn(f[j]));      // the operand's `.half()`
      }
    }
    float amax = 0.f;
    bool bad = false;
#pragma unroll
    for (int i = 0; i < U; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        bad |= !isfinite(v[i][j]);
        amax = fmaxf(amax, fabsf(v[i][j]));
      }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    bad = __any_sync(0xffffffffu, bad);
    int e = -15;
    while (e < 7 && amax > 448.f * __int_as_float((127 + e) << 23)) ++e;
    if (bad) e = 0;
    const float sc = __int_as_float((127 - e) << 23);                                   // 2^-e
    uint2 *dst = reinterpret_cast<uint2 *>(codes + r * C);
#pragma unroll
    for (int i = 0; i < U; ++i) {
      uint32_t w[2];
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        uint32_t lo, hi;
        {
          const float2 x = make_float2(fminf(fmaxf(v[i][4 * p] * sc, -448.f), 448.f),
                                       fminf(fmaxf(v[i][4 * p + 1] * sc, -448.f), 448.f));
          lo = __nv_cvt_float2_to_fp8x2(x, __NV_SATFINITE, __NV_E4M3);
        }
        {
          const float2 x = make_float2(fminf(fmaxf(v[i][4 * p + 2] * sc, -448.f), 448.f),
                                       fminf(fmaxf(v[i][4 * p + 3] * sc, -448.f), 448.f));
          hi = __nv_cvt_float2_to_fp8x2(x, __NV_SATFINITE, __NV_E4M3);
        }
        w[p] = bad ? 0x7f7f7f7fu : (lo | (hi << 16));
      }
      dst[lane + 32 * i] = make_uint2(w[0], w[1]);
    }
    if (lane == 0) row_exp[r] = (int8_t)e;
  }
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_search_workspace_bytes(int64_t n_scenes, int32_t nq, int32_t k) {
  if (n_scenes < 1 || nq < 1 || nq > OSB_SEARCH_MAX_QUERIES || k < 1 || k > OSB_SEARCH_MAX_K) return 0;
  return (size_t)SR_MAX_GRID * nq * k * 8 + (size_t)2 * n_scenes * nq * 8;
}

}  // extern "C"

// osb_search (row_exp NULL: fp16 rows) and osb_search_f8 (e4m3 codes and their exponents); fn names the entry point in
// the refusals
static int search_run(const char *fn, const void *rows_f16, const int8_t *row_exp, const int32_t *row_scene,
                      int64_t n_rows, int32_t c, const int64_t *scene_off_host, const int64_t *scene_off, int64_t n_scenes,
                      const void *queries_f16, int32_t nq, int32_t k, const float *threshold, void *top_score_f16,
                      int64_t *top_scene, int64_t *top_row, void *scene_max_f16, int64_t *scene_argmax,
                      int64_t *scene_count, void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(c == 512 || c == 768, "%s: feature width %d unsupported (OpenScene uses 512 / 768)", fn, c);
  OSB_CHECK(nq >= 1 && nq <= OSB_SEARCH_MAX_QUERIES, "%s: nq=%d outside 1..%d", fn, nq, OSB_SEARCH_MAX_QUERIES);
  OSB_CHECK(k >= 1 && k <= OSB_SEARCH_MAX_K, "%s: k=%d outside 1..%d", fn, k, OSB_SEARCH_MAX_K);
  OSB_CHECK(n_rows >= 1 && n_rows < (int64_t(1) << 31), "%s: N=%lld outside 1..2^31-1", fn, (long long)n_rows);
  OSB_CHECK(n_scenes >= 1 && n_scenes <= n_rows, "%s: %lld scenes for %lld rows", fn, (long long)n_scenes,
            (long long)n_rows);
  OSB_CHECK(rows_f16 && row_scene && scene_off_host && scene_off && queries_f16,
            "%s: NULL rows, row scenes, scene offsets or queries", fn);
  OSB_CHECK(top_score_f16 && top_scene && top_row && scene_max_f16 && scene_argmax,
            "%s: NULL top-k or per-scene output", fn);
  OSB_CHECK(scene_count == nullptr || threshold != nullptr, "%s: scene counts need a threshold", fn);
  OSB_CHECK(((uintptr_t)rows_f16 & 15) == 0 && ((uintptr_t)queries_f16 & 15) == 0,
            "%s: rows and queries must be 16-byte aligned", fn);
  OSB_CHECK(scene_off_host[0] == 0 && scene_off_host[n_scenes] == n_rows,
            "%s: scene offsets must run from 0 to N=%lld", fn, (long long)n_rows);
  for (int64_t s = 0; s < n_scenes; ++s)
    OSB_CHECK(scene_off_host[s] < scene_off_host[s + 1], "%s: scene offsets not strictly increasing at scene %lld", fn,
              (long long)s);
  const size_t need = osb_search_workspace_bytes(n_scenes, nq, k);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 7) == 0,
            "%s: 8-byte aligned workspace of %zu bytes required (got %zu)", fn, need, ws_bytes);

  const int64_t n_tiles = ceil_div(n_rows, MT_M);
  int dev = 0, sms = SR_MAX_GRID;
  OSB_CUDA(cudaGetDevice(&dev));
  OSB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = (int)std::min<int64_t>(n_tiles, std::min(sms, SR_MAX_GRID));

  SearchParams sp{};
  sp.a.feat = rows_f16; sp.a.feat_is_f16 = 1; sp.a.n_pts = n_rows; sp.a.C = c; sp.a.k_text = nq; sp.a.n_pass = 1;
  sp.row_scene = row_scene; sp.n = n_rows; sp.n_tiles = n_tiles; sp.nq = nq; sp.k = k; sp.row_exp = row_exp;
  sp.thr = scene_count ? threshold : nullptr;
  sp.lists = reinterpret_cast<uint64_t *>(ws);
  sp.scene_key = reinterpret_cast<unsigned long long *>(sp.lists + (size_t)SR_MAX_GRID * nq * k);
  sp.scene_cnt = sp.scene_key + (size_t)n_scenes * nq;
  OSB_CUDA(cudaMemsetAsync(sp.scene_key, 0, (size_t)2 * n_scenes * nq * 8, stream));

  CUtensorMap tmQ;
  if (make_tmap_2b(&tmQ, queries_f16, (uint64_t)c, (uint64_t)nq, MT_NW, 1)) return 1;
  const int NP = c / 64;
  const size_t smem = (size_t)NP * MT_M * 128 + MT_BSTAGES * MT_NW * 128 + 128 + MT_M * 4 + 1024;
  if (row_exp && NP == 12) {
    OSB_SMEM_ATTR_ONCE((k_search<12, false, true>), 227 * 1024);
    k_search<12, false, true><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  } else if (row_exp) {
    OSB_SMEM_ATTR_ONCE((k_search<8, false, true>), 227 * 1024);
    k_search<8, false, true><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  } else if (NP == 12) {
    OSB_SMEM_ATTR_ONCE(k_search<12>, 227 * 1024);
    k_search<12><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  } else {
    OSB_SMEM_ATTR_ONCE(k_search<8>, 227 * 1024);
    k_search<8><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  }
  OSB_LAUNCH_CHECK();
  const int scene_blocks = (int)std::min<int64_t>(ceil_div(n_scenes * nq, 256), 1024);
  k_search_finish<<<nq + scene_blocks, 256, (size_t)grid * k * 8, stream>>>(
      sp.lists, grid, nq, k, row_scene, scene_off, (__half *)top_score_f16, top_scene, top_row, sp.scene_key, sp.scene_cnt,
      n_scenes, (__half *)scene_max_f16, scene_argmax, scene_count);
  OSB_LAUNCH_CHECK();
  return 0;
}

extern "C" {

int osb_search(const void *rows_f16, const int32_t *row_scene, int64_t n_rows, int32_t c, const int64_t *scene_off_host,
               const int64_t *scene_off, int64_t n_scenes, const void *queries_f16, int32_t nq, int32_t k,
               const float *threshold, void *top_score_f16, int64_t *top_scene, int64_t *top_row, void *scene_max_f16,
               int64_t *scene_argmax, int64_t *scene_count, void *ws, size_t ws_bytes, void *stream) {
  return search_run("osb_search", rows_f16, nullptr, row_scene, n_rows, c, scene_off_host, scene_off, n_scenes,
                    queries_f16, nq, k, threshold, top_score_f16, top_scene, top_row, scene_max_f16, scene_argmax,
                    scene_count, ws, ws_bytes, stream);
}

int osb_search_f8(const void *codes_f8, const int8_t *row_exp, const int32_t *row_scene, int64_t n_rows, int32_t c,
                  const int64_t *scene_off_host, const int64_t *scene_off, int64_t n_scenes, const void *queries_f16,
                  int32_t nq, int32_t k, const float *threshold, void *top_score_f16, int64_t *top_scene, int64_t *top_row,
                  void *scene_max_f16, int64_t *scene_argmax, int64_t *scene_count, void *ws, size_t ws_bytes,
                  void *stream) {
  OSB_CHECK(row_exp != nullptr, "osb_search_f8: NULL row exponents");
  return search_run("osb_search_f8", codes_f8, row_exp, row_scene, n_rows, c, scene_off_host, scene_off, n_scenes,
                    queries_f16, nq, k, threshold, top_score_f16, top_scene, top_row, scene_max_f16, scene_argmax,
                    scene_count, ws, ws_bytes, stream);
}

size_t osb_search_hits_workspace_bytes(int64_t n_scenes, int32_t nq, int64_t n_hits) {
  if (n_scenes < 1 || nq < 1 || nq > OSB_SEARCH_MAX_QUERIES || n_hits < 1 || n_hits >= (int64_t(1) << 31)) return 0;
  // arrival keys 8, two payloads 4 + 4, arrival scores 2 (rounded up to 8 B per 4 hits), two [nq][S] arrays, sort histogram
  return (size_t)n_hits * 16 + (size_t)((n_hits + 3) / 4) * 8 + (size_t)2 * n_scenes * nq * 8 + radix_sort_ws_bytes(n_hits);
}

}  // extern "C"

// osb_search_hits (row_exp NULL: fp16 rows) and osb_search_hits_f8 (e4m3 codes and their exponents)
static int search_hits_run(const char *fn, const void *rows_f16, const int8_t *row_exp, const int32_t *row_scene,
                           int64_t n_rows, int32_t c, const int64_t *scene_off_host, int64_t n_scenes,
                           const void *queries_f16, int32_t nq, const float *threshold, const int64_t *scene_count,
                           int64_t n_hits, int64_t *hit_key, void *hit_score_f16, int32_t *status, void *ws,
                           size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(c == 512 || c == 768, "%s: feature width %d unsupported (OpenScene uses 512 / 768)", fn, c);
  OSB_CHECK(nq >= 1 && nq <= OSB_SEARCH_MAX_QUERIES, "%s: nq=%d outside 1..%d", fn, nq, OSB_SEARCH_MAX_QUERIES);
  OSB_CHECK(n_rows >= 1 && n_rows < (int64_t(1) << 31), "%s: N=%lld outside 1..2^31-1", fn, (long long)n_rows);
  OSB_CHECK(n_scenes >= 1 && n_scenes <= n_rows, "%s: %lld scenes for %lld rows", fn, (long long)n_scenes,
            (long long)n_rows);
  OSB_CHECK(n_hits >= 1 && n_hits < (int64_t(1) << 31), "%s: n_hits=%lld outside 1..2^31-1", fn,
            (long long)n_hits);
  OSB_CHECK(rows_f16 && row_scene && scene_off_host && queries_f16 && threshold && scene_count,
            "%s: NULL rows, row scenes, scene offsets, queries, threshold or scene counts", fn);
  OSB_CHECK(hit_key && hit_score_f16 && status, "%s: NULL hit list or status", fn);
  OSB_CHECK(((uintptr_t)rows_f16 & 15) == 0 && ((uintptr_t)queries_f16 & 15) == 0,
            "%s: rows and queries must be 16-byte aligned", fn);
  OSB_CHECK(((uintptr_t)hit_key & 7) == 0 && ((uintptr_t)hit_score_f16 & 1) == 0 && ((uintptr_t)status & 3) == 0,
            "%s: misaligned hit list or status", fn);
  OSB_CHECK(scene_off_host[0] == 0 && scene_off_host[n_scenes] == n_rows,
            "%s: scene offsets must run from 0 to N=%lld", fn, (long long)n_rows);
  for (int64_t s = 0; s < n_scenes; ++s)
    OSB_CHECK(scene_off_host[s] < scene_off_host[s + 1],
              "%s: scene offsets not strictly increasing at scene %lld", fn, (long long)s);
  const size_t need = osb_search_hits_workspace_bytes(n_scenes, nq, n_hits);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 7) == 0,
            "%s: 8-byte aligned workspace of %zu bytes required (got %zu)", fn, need, ws_bytes);

  uint8_t *w = reinterpret_cast<uint8_t *>(ws);
  uint64_t *keys_a = reinterpret_cast<uint64_t *>(w);                       w += (size_t)n_hits * 8;
  int32_t *vals_a = reinterpret_cast<int32_t *>(w);                         w += (size_t)n_hits * 4;
  int32_t *vals_b = reinterpret_cast<int32_t *>(w);                         w += (size_t)n_hits * 4;
  __half *score_a = reinterpret_cast<__half *>(w);                          w += (size_t)((n_hits + 3) / 4) * 8;
  unsigned long long *cursor = reinterpret_cast<unsigned long long *>(w);   w += (size_t)n_scenes * nq * 8;
  unsigned long long *seg_end = reinterpret_cast<unsigned long long *>(w);  w += (size_t)n_scenes * nq * 8;
  void *sort_ws = w;

  k_hit_segments<<<1, 1024, 0, stream>>>(scene_count, n_scenes, nq, n_hits, cursor, seg_end, status);
  OSB_LAUNCH_CHECK();

  const int64_t n_tiles = ceil_div(n_rows, MT_M);
  int dev = 0, sms = SR_MAX_GRID;
  OSB_CUDA(cudaGetDevice(&dev));
  OSB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int grid = (int)std::min<int64_t>(n_tiles, std::min(sms, SR_MAX_GRID));
  SearchParams sp{};
  sp.a.feat = rows_f16; sp.a.feat_is_f16 = 1; sp.a.n_pts = n_rows; sp.a.C = c; sp.a.k_text = nq; sp.a.n_pass = 1;
  sp.row_scene = row_scene; sp.n = n_rows; sp.n_tiles = n_tiles; sp.nq = nq; sp.k = 1;
  sp.thr = threshold; sp.row_exp = row_exp;
  sp.n_scenes = n_scenes; sp.cursor = cursor; sp.seg_end = seg_end; sp.hit_key = keys_a; sp.hit_score = score_a;
  sp.status = status;
  CUtensorMap tmQ;
  if (make_tmap_2b(&tmQ, queries_f16, (uint64_t)c, (uint64_t)nq, MT_NW, 1)) return 1;
  const int NP = c / 64;
  const size_t smem = (size_t)NP * MT_M * 128 + MT_BSTAGES * MT_NW * 128 + 128 + MT_M * 4 + 1024;
  if (row_exp && NP == 12) {
    OSB_SMEM_ATTR_ONCE((k_search<12, true, true>), 227 * 1024);
    k_search<12, true, true><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  } else if (row_exp) {
    OSB_SMEM_ATTR_ONCE((k_search<8, true, true>), 227 * 1024);
    k_search<8, true, true><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  } else if (NP == 12) {
    OSB_SMEM_ATTR_ONCE((k_search<12, true>), 227 * 1024);
    k_search<12, true><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  } else {
    OSB_SMEM_ATTR_ONCE((k_search<8, true>), 227 * 1024);
    k_search<8, true><<<grid, MT_THREADS, smem, stream>>>(tmQ, sp);
  }
  OSB_LAUNCH_CHECK();

  // canonical order: stable sort by (query << 32) | global row, distinct per hit (bits 0..38: q < 96, row < 2^31)
  uint64_t *keys_out = reinterpret_cast<uint64_t *>(hit_key);
  const int where = radix_sort_pairs(keys_a, vals_a, keys_out, vals_b, nullptr, n_hits, 0, 39, sort_ws, stream);
  OSB_CHECK(where >= 0, "%s: sort launch failed", fn);
  const int32_t *slot = where ? vals_b : vals_a;
  if (where == 0) OSB_CUDA(cudaMemcpyAsync(keys_out, keys_a, (size_t)n_hits * 8, cudaMemcpyDeviceToDevice, stream));
  const int blocks = (int)std::min<int64_t>(ceil_div(std::max<int64_t>(n_hits, n_scenes * nq), 256), 4096);
  k_hit_finish<<<blocks, 256, 0, stream>>>(cursor, seg_end, n_scenes * nq, slot, score_a, n_hits,
                                           (__half *)hit_score_f16, status);
  OSB_LAUNCH_CHECK();
  return 0;
}

extern "C" {

int osb_search_hits(const void *rows_f16, const int32_t *row_scene, int64_t n_rows, int32_t c, const int64_t *scene_off_host,
                    int64_t n_scenes, const void *queries_f16, int32_t nq, const float *threshold,
                    const int64_t *scene_count, int64_t n_hits, int64_t *hit_key, void *hit_score_f16, int32_t *status,
                    void *ws, size_t ws_bytes, void *stream) {
  return search_hits_run("osb_search_hits", rows_f16, nullptr, row_scene, n_rows, c, scene_off_host, n_scenes, queries_f16,
                         nq, threshold, scene_count, n_hits, hit_key, hit_score_f16, status, ws, ws_bytes, stream);
}

int osb_search_hits_f8(const void *codes_f8, const int8_t *row_exp, const int32_t *row_scene, int64_t n_rows, int32_t c,
                       const int64_t *scene_off_host, int64_t n_scenes, const void *queries_f16, int32_t nq,
                       const float *threshold, const int64_t *scene_count, int64_t n_hits, int64_t *hit_key,
                       void *hit_score_f16, int32_t *status, void *ws, size_t ws_bytes, void *stream) {
  OSB_CHECK(row_exp != nullptr, "osb_search_hits_f8: NULL row exponents");
  return search_hits_run("osb_search_hits_f8", codes_f8, row_exp, row_scene, n_rows, c, scene_off_host, n_scenes,
                         queries_f16, nq, threshold, scene_count, n_hits, hit_key, hit_score_f16, status, ws, ws_bytes,
                         stream);
}

int osb_index_quantize_f8(const void *rows, int32_t rows_are_f16, int64_t n, int32_t c, void *codes_out, int8_t *exp_out,
                          void *stream) {
  OSB_CHECK(c == 512 || c == 768, "osb_index_quantize_f8: feature width %d unsupported (OpenScene uses 512 / 768)", c);
  OSB_CHECK(n >= 1 && n < (int64_t(1) << 31), "osb_index_quantize_f8: N=%lld outside 1..2^31-1", (long long)n);
  OSB_CHECK(rows && codes_out && exp_out, "osb_index_quantize_f8: NULL rows, codes or exponents");
  OSB_CHECK(((uintptr_t)rows & 15) == 0 && ((uintptr_t)codes_out & 15) == 0,
            "osb_index_quantize_f8: rows and codes must be 16-byte aligned");
  const int blocks = (int)std::min<int64_t>(ceil_div(n, 8), 132 * 16);
  if (c == 768)
    k_index_quantize_f8<12><<<blocks, 256, 0, (cudaStream_t)stream>>>(rows, rows_are_f16 != 0, n,
                                                                       (uint8_t *)codes_out, exp_out);
  else
    k_index_quantize_f8<8><<<blocks, 256, 0, (cudaStream_t)stream>>>(rows, rows_are_f16 != 0, n, (uint8_t *)codes_out,
                                                                      exp_out);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
