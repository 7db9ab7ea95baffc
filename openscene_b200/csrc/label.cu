// Class counts and class hit lists of a labelled scene index (DESIGN.md, "Label contract").
//
// SceneIndex.label gives every row r its label row_label[r] (the top-1 column of osb_match_topk against a vocabulary of K
// classes) and that column's fp16 score row_label_score[r].  A query is a host list of m distinct classes; slot j stands for
// classes[j], through a device table [K] (class -> slot or -1) built from the list in the workspace.
//
//   osb_label_counts  counts[s, j] = rows of scene s labelled classes[j] (with a threshold: whose score is not NaN and
//                     float(score) >= thr[j]).  One pass over the rows (14 B per row).  A block owns a 4096-row chunk
//                     and keeps a shared-memory histogram of the (scene, slot) pairs of its chunk, flushed with integer
//                     atomicAdd: the common classes of a scene (floor, wall) cost one global atomic per block, not per
//                     row.  Pairs past the shared capacity (many tiny scenes times many slots) go to global atomics.
//   osb_label_hits    the hit list of one slice of at most 96 slots, in the layout osb_search_hits writes and osb_regions
//                     takes: hit_key = (slot << 32) | global row ascending, hit_score the label score.  The rows already
//                     are in global-row order, so an order-preserving compaction replaces the radix sort: per block and
//                     slot a hit count, an exclusive scan of those over the blocks from the slot's base (the segment
//                     bases of k_hit_segments), and a block-ordered write.  Every hit is checked to land inside its
//                     (slot, scene) segment, and every slot to receive exactly its counted hits; a miss sets
//                     OSB_REGIONS_ST_COUNT.
//
// Integer atomics only: two calls give the same bits.
#include "common.cuh"
#include <algorithm>

namespace osb {

constexpr int LB_THREADS = 256;
constexpr int LB_CHUNK = 4096;           // rows per block
constexpr int LB_SMEM_PAIRS = 8192;      // shared (scene, slot) counters per block (32 KB)
constexpr int LB_MAX_SLOTS = 96;         // slots of one osb_label_hits slice (OSB_SEARCH_MAX_QUERIES)

// segments of a hit list in (slot, scene) order from its counts [S][m] (search.cu)
int hit_segments_run(const int64_t *scene_count, int64_t n_scenes, int nq, int64_t n_hits, unsigned long long *cursor,
                     unsigned long long *seg_end, int *status, cudaStream_t stream);

// table[k] = slot of class k, or -1 (the caller set the table to -1)
__global__ void k_label_table(const int64_t *__restrict__ classes, int m, int32_t *__restrict__ table) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < m; j += gridDim.x * blockDim.x) table[classes[j]] = j;
}

// the slot of row r when it counts, else -1
__device__ __forceinline__ int label_slot(const int64_t *__restrict__ row_label, const __half *__restrict__ row_score,
                                          const int32_t *__restrict__ table, int k_text, const float *__restrict__ thr,
                                          int64_t r) {
  const int64_t y = __ldg(row_label + r);
  if ((uint64_t)y >= (uint64_t)k_text) return -1;
  const int j = __ldg(table + y);
  if (j < 0 || thr == nullptr) return j;
  const float s = __half2float(__ldg(row_score + r));
  return s >= __ldg(thr + j) ? j : -1;                        // NaN never passes
}

__global__ void __launch_bounds__(LB_THREADS)
k_label_counts(const int64_t *__restrict__ row_label, const __half *__restrict__ row_score,
               const int32_t *__restrict__ row_scene, int64_t n, const int32_t *__restrict__ table, int k_text, int m,
               const float *__restrict__ thr, unsigned long long *__restrict__ counts) {
  __shared__ uint32_t s_cnt[LB_SMEM_PAIRS];
  const int64_t a = (int64_t)blockIdx.x * LB_CHUNK, b = std::min<int64_t>(n, a + LB_CHUNK);
  const int s0 = __ldg(row_scene + a), s1 = __ldg(row_scene + b - 1);
  const int64_t pairs = std::min<int64_t>((int64_t)(s1 - s0 + 1) * m, LB_SMEM_PAIRS);
  for (int64_t i = threadIdx.x; i < pairs; i += LB_THREADS) s_cnt[i] = 0;
  __syncthreads();
  for (int64_t r = a + threadIdx.x; r < b; r += LB_THREADS) {
    const int j = label_slot(row_label, row_score, table, k_text, thr, r);
    if (j < 0) continue;
    const int s = __ldg(row_scene + r);
    const int64_t e = (int64_t)(s - s0) * m + j;
    if (e < pairs) atomicAdd(s_cnt + e, 1u);
    else atomicAdd(counts + (int64_t)s * m + j, 1ull);
  }
  __syncthreads();
  for (int64_t i = threadIdx.x; i < pairs; i += LB_THREADS)
    if (s_cnt[i]) atomicAdd(counts + (int64_t)s0 * m + i, (unsigned long long)s_cnt[i]);
}

// bcnt[j][blk]: the hits of slot j in block blk's chunk
__global__ void __launch_bounds__(LB_THREADS)
k_label_block_counts(const int64_t *__restrict__ row_label, const __half *__restrict__ row_score, int64_t n,
                     const int32_t *__restrict__ table, int k_text, int m, const float *__restrict__ thr,
                     uint32_t *__restrict__ bcnt) {
  __shared__ uint32_t s_cnt[LB_MAX_SLOTS];
  for (int j = threadIdx.x; j < m; j += LB_THREADS) s_cnt[j] = 0;
  __syncthreads();
  const int64_t a = (int64_t)blockIdx.x * LB_CHUNK, b = std::min<int64_t>(n, a + LB_CHUNK);
  for (int64_t r = a + threadIdx.x; r < b; r += LB_THREADS) {
    const int j = label_slot(row_label, row_score, table, k_text, thr, r);
    if (j >= 0) atomicAdd(s_cnt + j, 1u);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < m; j += LB_THREADS) bcnt[(int64_t)j * gridDim.x + blockIdx.x] = s_cnt[j];
}

// one block per slot j: boff[j][blk] = the slot's base (cursor[j][0]) + exclusive scan of bcnt[j][:]; the slot's total must
// equal its counts' sum
__global__ void __launch_bounds__(1024)
k_label_block_scan(const uint32_t *__restrict__ bcnt, int64_t nblk, const int64_t *__restrict__ counts, int64_t n_scenes,
                   int m, const unsigned long long *__restrict__ cursor, unsigned long long *__restrict__ boff,
                   int *status) {
  __shared__ unsigned long long s_part[1024], s_total, s_want;
  const int j = blockIdx.x;
  const uint32_t *c = bcnt + (int64_t)j * nblk;
  const int64_t per = (nblk + 1023) / 1024;
  const int64_t a = std::min<int64_t>(nblk, per * threadIdx.x), b = std::min<int64_t>(nblk, a + per);
  unsigned long long t = 0;
  for (int64_t i = a; i < b; ++i) t += c[i];
  s_part[threadIdx.x] = t;
  if (threadIdx.x == 0) s_want = 0;
  __syncthreads();
  unsigned long long want = 0;
  for (int64_t s = threadIdx.x; s < n_scenes; s += 1024) want += (unsigned long long)counts[s * m + j];
  if (want) atomicAdd(&s_want, want);
  if (threadIdx.x == 0) {
    unsigned long long run = 0;
    for (int i = 0; i < 1024; ++i) { const unsigned long long v = s_part[i]; s_part[i] = run; run += v; }
    s_total = run;
  }
  __syncthreads();
  if (threadIdx.x == 0 && s_want != s_total) atomicOr(status, OSB_REGIONS_ST_COUNT);
  unsigned long long run = cursor[(int64_t)j * n_scenes] + s_part[threadIdx.x];
  for (int64_t i = a; i < b; ++i) {
    boff[(int64_t)j * nblk + i] = run;
    run += c[i];
  }
}

// the block's hits in row order: per round of 256 rows, a thread's position among the hits of its slot is the block's
// running count of the slot, plus the slot's hits of the lower warps, plus its rank among the lanes of its warp
__global__ void __launch_bounds__(LB_THREADS)
k_label_emit(const int64_t *__restrict__ row_label, const __half *__restrict__ row_score,
             const int32_t *__restrict__ row_scene, int64_t n, const int32_t *__restrict__ table, int k_text, int m,
             const float *__restrict__ thr, int64_t n_scenes, const unsigned long long *__restrict__ boff,
             const unsigned long long *__restrict__ cursor, const unsigned long long *__restrict__ seg_end,
             int64_t n_hits, int64_t *__restrict__ hit_key, __half *__restrict__ hit_score, int *status) {
  constexpr int W = LB_THREADS / 32;
  __shared__ uint32_t s_wc[W][LB_MAX_SLOTS];
  __shared__ unsigned long long s_run[LB_MAX_SLOTS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = threadIdx.x; j < m; j += LB_THREADS) s_run[j] = boff[(int64_t)j * gridDim.x + blockIdx.x];
  const int64_t a = (int64_t)blockIdx.x * LB_CHUNK, b = std::min<int64_t>(n, a + LB_CHUNK);
  bool bad = false;
  for (int64_t r0 = a; r0 < b; r0 += LB_THREADS) {
    __syncthreads();      // the previous round's readers of s_wc are done
    for (int i = threadIdx.x; i < W * m; i += LB_THREADS) s_wc[i / m][i % m] = 0;
    __syncthreads();
    const int64_t r = r0 + threadIdx.x;
    const int j = r < b ? label_slot(row_label, row_score, table, k_text, thr, r) : -1;
    const uint32_t peers = __match_any_sync(0xffffffffu, j);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (j >= 0 && rank == 0) s_wc[warp][j] = __popc(peers);
    __syncthreads();
    if (j >= 0) {
      unsigned long long pos = s_run[j] + rank;
      for (int w = 0; w < warp; ++w) pos += s_wc[w][j];
      const int64_t seg = (int64_t)j * n_scenes + __ldg(row_scene + r);
      if (pos < cursor[seg] || pos >= seg_end[seg] || pos >= (unsigned long long)n_hits) {
        bad = true;
      } else {
        hit_key[pos] = ((int64_t)j << 32) | r;
        hit_score[pos] = row_score[r];
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += LB_THREADS) {
      unsigned long long t = 0;
      for (int w = 0; w < W; ++w) t += s_wc[w][i];
      s_run[i] += t;
    }
  }
  if (bad) atomicOr(status, OSB_REGIONS_ST_COUNT);
}

// the shared refusals of both entry points
static int label_args(const char *fn, const int64_t *row_label, const void *row_score_f16, const int32_t *row_scene,
                      int64_t n_rows, int64_t n_scenes, int32_t k_text, const int64_t *classes_host, int32_t m) {
  OSB_CHECK(k_text >= 1 && k_text <= OSB_MATCH_TOPK_MAX_TEXT, "%s: K=%d outside 1..%d", fn, k_text,
            OSB_MATCH_TOPK_MAX_TEXT);
  OSB_CHECK(m >= 1 && m <= k_text, "%s: m=%d classes outside 1..K=%d", fn, m, k_text);
  OSB_CHECK(n_rows >= 1 && n_rows < (int64_t(1) << 31), "%s: N=%lld outside 1..2^31-1", fn, (long long)n_rows);
  OSB_CHECK(n_scenes >= 1 && n_scenes <= n_rows, "%s: %lld scenes for %lld rows", fn, (long long)n_scenes,
            (long long)n_rows);
  OSB_CHECK(row_label && row_score_f16 && row_scene && classes_host, "%s: NULL labels, label scores, row scenes or classes",
            fn);
  OSB_CHECK(((uintptr_t)row_label & 7) == 0 && ((uintptr_t)row_score_f16 & 1) == 0 && ((uintptr_t)row_scene & 3) == 0,
            "%s: misaligned labels, label scores or row scenes", fn);
  for (int32_t j = 0; j < m; ++j)
    OSB_CHECK(classes_host[j] >= 0 && classes_host[j] < k_text, "%s: class %lld (slot %d) outside 0..K-1=%d", fn,
              (long long)classes_host[j], j, k_text - 1);
  // duplicates: a sorted copy
  int64_t *sorted = new int64_t[m];
  std::copy(classes_host, classes_host + m, sorted);
  std::sort(sorted, sorted + m);
  int64_t dup = -1;
  for (int32_t j = 1; j < m && dup < 0; ++j)
    if (sorted[j] == sorted[j - 1]) dup = sorted[j];
  delete[] sorted;
  OSB_CHECK(dup < 0, "%s: class %lld listed twice", fn, (long long)dup);
  return 0;
}

static size_t table_bytes(int32_t k_text, int32_t m) {
  return (size_t)ceil_div(k_text, 2) * 8 + (size_t)m * 8;
}

// the class -> slot table at the start of the workspace: the host list is copied in (no wait on the device), the table set
// to -1 and scattered
static int label_table(const int64_t *classes_host, int32_t m, int32_t k_text, void *ws, int32_t **table,
                       cudaStream_t stream) {
  *table = reinterpret_cast<int32_t *>(ws);
  int64_t *cls = reinterpret_cast<int64_t *>(reinterpret_cast<uint8_t *>(ws) + (size_t)ceil_div(k_text, 2) * 8);
  OSB_CUDA(cudaMemcpyAsync(cls, classes_host, (size_t)m * 8, cudaMemcpyHostToDevice, stream));
  OSB_CUDA(cudaMemsetAsync(*table, 0xff, (size_t)k_text * 4, stream));
  k_label_table<<<(unsigned)std::min<int64_t>(ceil_div(m, 256), 1024), 256, 0, stream>>>(cls, m, *table);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_label_counts_workspace_bytes(int32_t k_text, int32_t m) {
  if (k_text < 1 || k_text > OSB_MATCH_TOPK_MAX_TEXT || m < 1 || m > k_text) return 0;
  return table_bytes(k_text, m);
}

int osb_label_counts(const int64_t *row_label, const void *row_score_f16, const int32_t *row_scene, int64_t n_rows,
                     int64_t n_scenes, int32_t k_text, const int64_t *classes_host, int32_t m, const float *threshold,
                     int64_t *counts, void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (label_args("osb_label_counts", row_label, row_score_f16, row_scene, n_rows, n_scenes, k_text, classes_host, m))
    return 1;
  OSB_CHECK(n_scenes * m <= OSB_LABEL_MAX_COUNTS, "osb_label_counts: %lld scenes x %d classes exceed %d counts",
            (long long)n_scenes, m, OSB_LABEL_MAX_COUNTS);
  OSB_CHECK(counts != nullptr && ((uintptr_t)counts & 7) == 0, "osb_label_counts: NULL or misaligned counts");
  OSB_CHECK(threshold == nullptr || ((uintptr_t)threshold & 3) == 0, "osb_label_counts: misaligned threshold");
  const size_t need = osb_label_counts_workspace_bytes(k_text, m);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 7) == 0,
            "osb_label_counts: 8-byte aligned workspace of %zu bytes required (got %zu)", need, ws_bytes);
  int32_t *table;
  if (label_table(classes_host, m, k_text, ws, &table, stream)) return 1;
  OSB_CUDA(cudaMemsetAsync(counts, 0, (size_t)n_scenes * m * 8, stream));
  k_label_counts<<<(unsigned)ceil_div(n_rows, LB_CHUNK), LB_THREADS, 0, stream>>>(
      row_label, (const __half *)row_score_f16, row_scene, n_rows, table, k_text, m, threshold,
      reinterpret_cast<unsigned long long *>(counts));
  OSB_LAUNCH_CHECK();
  return 0;
}

size_t osb_label_hits_workspace_bytes(int32_t k_text, int64_t n_rows, int64_t n_scenes, int32_t m) {
  if (k_text < 1 || k_text > OSB_MATCH_TOPK_MAX_TEXT || m < 1 || m > std::min(k_text, LB_MAX_SLOTS) || n_rows < 1 ||
      n_rows >= (int64_t(1) << 31) || n_scenes < 1 || n_scenes > n_rows)
    return 0;
  const int64_t nblk = ceil_div(n_rows, LB_CHUNK);
  // table, cursor and seg_end [m][S], block offsets [m][nblk] (8 B), block counts [m][nblk] (4 B, rounded up)
  return table_bytes(k_text, m) + (size_t)2 * m * n_scenes * 8 + (size_t)m * nblk * 8 + (size_t)ceil_div(m * nblk, 2) * 8;
}

int osb_label_hits(const int64_t *row_label, const void *row_score_f16, const int32_t *row_scene, int64_t n_rows,
                   int64_t n_scenes, int32_t k_text, const int64_t *classes_host, int32_t m, const float *threshold,
                   const int64_t *counts, int64_t n_hits, int64_t *hit_key, void *hit_score_f16, int32_t *status, void *ws,
                   size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (label_args("osb_label_hits", row_label, row_score_f16, row_scene, n_rows, n_scenes, k_text, classes_host, m))
    return 1;
  OSB_CHECK(m <= LB_MAX_SLOTS, "osb_label_hits: m=%d classes above %d per call", m, LB_MAX_SLOTS);
  OSB_CHECK(n_hits >= 1 && n_hits < (int64_t(1) << 31), "osb_label_hits: n_hits=%lld outside 1..2^31-1",
            (long long)n_hits);
  OSB_CHECK(threshold && counts && hit_key && hit_score_f16 && status,
            "osb_label_hits: NULL threshold, counts, hit list or status");
  OSB_CHECK(((uintptr_t)threshold & 3) == 0 && ((uintptr_t)counts & 7) == 0 && ((uintptr_t)hit_key & 7) == 0 &&
                ((uintptr_t)hit_score_f16 & 1) == 0 && ((uintptr_t)status & 3) == 0,
            "osb_label_hits: misaligned threshold, counts, hit list or status");
  const size_t need = osb_label_hits_workspace_bytes(k_text, n_rows, n_scenes, m);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 7) == 0,
            "osb_label_hits: 8-byte aligned workspace of %zu bytes required (got %zu)", need, ws_bytes);
  const int64_t nblk = ceil_div(n_rows, LB_CHUNK);
  uint8_t *w = reinterpret_cast<uint8_t *>(ws) + table_bytes(k_text, m);
  unsigned long long *cursor = reinterpret_cast<unsigned long long *>(w);   w += (size_t)m * n_scenes * 8;
  unsigned long long *seg_end = reinterpret_cast<unsigned long long *>(w);  w += (size_t)m * n_scenes * 8;
  unsigned long long *boff = reinterpret_cast<unsigned long long *>(w);     w += (size_t)m * nblk * 8;
  uint32_t *bcnt = reinterpret_cast<uint32_t *>(w);
  int32_t *table;
  if (label_table(classes_host, m, k_text, ws, &table, stream)) return 1;
  if (hit_segments_run(counts, n_scenes, m, n_hits, cursor, seg_end, status, stream)) return 1;
  const __half *score = (const __half *)row_score_f16;
  k_label_block_counts<<<(unsigned)nblk, LB_THREADS, 0, stream>>>(row_label, score, n_rows, table, k_text, m, threshold,
                                                                   bcnt);
  OSB_LAUNCH_CHECK();
  k_label_block_scan<<<m, 1024, 0, stream>>>(bcnt, nblk, counts, n_scenes, m, cursor, boff, status);
  OSB_LAUNCH_CHECK();
  k_label_emit<<<(unsigned)nblk, LB_THREADS, 0, stream>>>(row_label, score, row_scene, n_rows, table, k_text, m, threshold,
                                                          n_scenes, boff, cursor, seg_end, n_hits, hit_key,
                                                          (__half *)hit_score_f16, status);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
