// Sharded scene index (DESIGN.md, "Sharded index contract"): the scenes of one database spread over the ranks of a
// process group, each rank searching its own SceneIndex with k_search and osb_regions; these kernels merge the small
// per-rank results into the answer of one index holding every scene in ascending global id.
//
//   k_shard_keys        a rank's decoded (score, local scene, row) -> 64-bit global key and global scene id.  Bits 48-63
//                       the score's order (search_key's map: -0 as +0, inf above every finite value), bits 0-47 ~global
//                       row, global row = base[global id] + row; NaN and padding slots (scene -1) have key 0
//   k_shard_merge       per query the m best of world x m keys, as source positions w * m + j.  Each rank's list is
//                       already in descending key order (a rank keeps its scenes in ascending global id, so its local
//                       row order is the global row order), so a k-way merge does it: m rounds, each one warp argmax
//                       over the heads of at most 64 lists, no shared-memory sort of world x m keys.  Keys of real
//                       entries are distinct (one global row each); ties among padding keys go to the lower list, so
//                       the winners are distinct positions
//   k_shard_hit_*       the gathered hit lists in (query, global row) order by the stable radix sort of sortscan.cuh,
//                       and each hit's local region rank mapped to its rank in the merged list through the winner table
// Integer work only: two calls give the same bits on any stream.
#include "sortscan.cuh"
#include <climits>

namespace osb {

constexpr uint64_t SH_ROW_MASK = (uint64_t(1) << 48) - 1;

__global__ void k_shard_keys(const __half *__restrict__ score, const int64_t *__restrict__ scene,
                             const int64_t *__restrict__ row, int64_t n, const int64_t *__restrict__ gid, int64_t n_local,
                             const int64_t *__restrict__ base, int64_t n_global, int64_t *key, int64_t *gscene) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t s = scene[i];
    const int64_t g = (s >= 0 && s < n_local) ? gid[s] : -1;
    const uint32_t b = __half_as_ushort(score[i]);
    uint64_t k = 0;
    if (g >= 0 && g < n_global && (b & 0x7fffu) <= 0x7c00u) {
      const uint32_t u = b == 0x8000u ? 0x8000u : (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
      k = ((uint64_t)u << 48) | (~(uint64_t)(base[g] + row[i]) & SH_ROW_MASK);
    }
    key[i] = (int64_t)k;
    gscene[i] = g;
  }
}

// block q, one warp: lane l owns the heads of lists l and l + 32
__global__ void __launch_bounds__(32) k_shard_merge(const int64_t *__restrict__ keys, int world, int nq, int m,
                                                    int64_t *winners) {
  const int q = blockIdx.x, lane = threadIdx.x;
  int head[2] = {0, 0};
  for (int j = 0; j < m; ++j) {
    unsigned long long bk = 0;
    int bl = INT_MAX;                                  // no candidate
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int l = lane + 32 * h;
      if (l < world && head[h] < m) {
        const unsigned long long v = (unsigned long long)keys[((size_t)l * nq + q) * m + head[h]];
        if (bl == INT_MAX || v > bk) { bk = v; bl = l; }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long ok = __shfl_xor_sync(0xffffffffu, bk, o);
      const int ol = __shfl_xor_sync(0xffffffffu, bl, o);
      if (ol != INT_MAX && (bl == INT_MAX || ok > bk || (ok == bk && ol < bl))) { bk = ok; bl = ol; }
    }
    // every lane holds the winning list bl; its owner advances that head
    const int h = bl >> 5, wl = bl & 31;
    const int pos = __shfl_sync(0xffffffffu, h ? head[1] : head[0], wl);
    if (lane == 0) winners[(size_t)q * m + j] = (int64_t)bl * m + pos;
    if (lane == wl) ++head[h];
  }
}

__global__ void k_shard_hit_keys(const int64_t *__restrict__ query, const int64_t *__restrict__ grow, int64_t n,
                                 uint64_t *key) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) key[i] = ((uint64_t)query[i] << 48) | ((uint64_t)grow[i] & SH_ROW_MASK);
}

// sorted position i: the source hit, and its region's rank in the merged list (-1 when the region is not in it)
__global__ void k_shard_hit_finish(const int32_t *__restrict__ perm, int64_t n, const int64_t *__restrict__ query,
                                   const int64_t *__restrict__ rank, const int64_t *__restrict__ region,
                                   const int64_t *__restrict__ winners, int R, int64_t *order, int64_t *region_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = perm[i];
  const int64_t r = region[p];
  int64_t out = -1;
  if (r >= 0 && r < R) {
    const int64_t want = rank[p] * R + r, *w = winners + (size_t)query[p] * R;
    for (int j = 0; j < R; ++j)
      if (w[j] == want) { out = j; break; }
  }
  order[i] = p;
  region_out[i] = out;
}

static inline int sh_bits_for(uint64_t n) {   // bits of the largest value below n
  int b = 0;
  while (b < 64 && (n - 1) >> b) ++b;
  return b;
}

}  // namespace osb

using namespace osb;

extern "C" {

int osb_shard_keys(const void *score_f16, const int64_t *scene, const int64_t *row, int64_t n, const int64_t *scene_gid,
                   int64_t n_local, const int64_t *row_base, int64_t n_global, int64_t n_rows_global, int64_t *key,
                   int64_t *global_scene, void *stream) {
  OSB_CHECK(n >= 1 && n < (int64_t(1) << 40), "osb_shard_keys: n=%lld outside 1..2^40-1", (long long)n);
  OSB_CHECK(n_local >= 0 && n_global >= 1 && n_local <= n_global, "osb_shard_keys: %lld local scenes of %lld",
            (long long)n_local, (long long)n_global);
  OSB_CHECK(n_rows_global >= n_global && n_rows_global < (int64_t(1) << 48),
            "osb_shard_keys: %lld rows over the group outside %lld..2^48-1", (long long)n_rows_global,
            (long long)n_global);
  OSB_CHECK(score_f16 && scene && row && row_base && key && global_scene && (n_local == 0 || scene_gid),
            "osb_shard_keys: NULL results, directory or output");
  OSB_CHECK(((uintptr_t)score_f16 & 1) == 0 && ((uintptr_t)scene & 7) == 0 && ((uintptr_t)row & 7) == 0 &&
                ((uintptr_t)scene_gid & 7) == 0 && ((uintptr_t)row_base & 7) == 0 && ((uintptr_t)key & 7) == 0 &&
                ((uintptr_t)global_scene & 7) == 0,
            "osb_shard_keys: misaligned results, directory or output");
  const int blocks = (int)std::min<int64_t>(ceil_div(n, 256), 1024);
  k_shard_keys<<<blocks, 256, 0, (cudaStream_t)stream>>>((const __half *)score_f16, scene, row, n, scene_gid, n_local,
                                                         row_base, n_global, key, global_scene);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_shard_merge(const int64_t *keys, int32_t world, int32_t nq, int32_t m, int64_t *winners, void *stream) {
  OSB_CHECK(world >= 1 && world <= OSB_SHARD_MAX_WORLD, "osb_shard_merge: world=%d outside 1..%d", world,
            OSB_SHARD_MAX_WORLD);
  OSB_CHECK(nq >= 1 && nq <= OSB_SHARD_MAX_QUERIES, "osb_shard_merge: nq=%d outside 1..%d", nq, OSB_SHARD_MAX_QUERIES);
  OSB_CHECK(m >= 1 && m <= OSB_SHARD_MAX_M, "osb_shard_merge: m=%d outside 1..%d", m, OSB_SHARD_MAX_M);
  OSB_CHECK(keys && winners, "osb_shard_merge: NULL keys or winners");
  OSB_CHECK(((uintptr_t)keys & 7) == 0 && ((uintptr_t)winners & 7) == 0, "osb_shard_merge: misaligned keys or winners");
  k_shard_merge<<<nq, 32, 0, (cudaStream_t)stream>>>(keys, world, nq, m, winners);
  OSB_LAUNCH_CHECK();
  return 0;
}

size_t osb_shard_hits_workspace_bytes(int64_t n_hits) {
  if (n_hits < 1 || n_hits >= (int64_t(1) << 31)) return 0;
  // two key buffers 8 + 8, two payloads 4 + 4 (each rounded to 256 B), sort histogram
  return (size_t)2 * (((size_t)n_hits * 8 + 255) & ~size_t(255)) + (size_t)2 * (((size_t)n_hits * 4 + 255) & ~size_t(255)) +
         radix_sort_ws_bytes(n_hits);
}

int osb_shard_hits(const int64_t *hit_query, const int64_t *hit_grow, const int64_t *hit_rank, const int64_t *hit_region,
                   int64_t n_hits, int32_t world, int32_t nq, int32_t R, const int64_t *winners, int64_t *order,
                   int64_t *region_out, void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(world >= 1 && world <= OSB_SHARD_MAX_WORLD, "osb_shard_hits: world=%d outside 1..%d", world,
            OSB_SHARD_MAX_WORLD);
  OSB_CHECK(nq >= 1 && nq <= OSB_SHARD_MAX_QUERIES, "osb_shard_hits: nq=%d outside 1..%d", nq, OSB_SHARD_MAX_QUERIES);
  OSB_CHECK(R >= 1 && R <= OSB_SHARD_MAX_M, "osb_shard_hits: R=%d outside 1..%d", R, OSB_SHARD_MAX_M);
  OSB_CHECK(n_hits >= 1 && n_hits < (int64_t(1) << 31), "osb_shard_hits: n_hits=%lld outside 1..2^31-1",
            (long long)n_hits);
  OSB_CHECK(hit_query && hit_grow && hit_rank && hit_region && winners && order && region_out,
            "osb_shard_hits: NULL hit list, winners or output");
  OSB_CHECK(((uintptr_t)hit_query & 7) == 0 && ((uintptr_t)hit_grow & 7) == 0 && ((uintptr_t)hit_rank & 7) == 0 &&
                ((uintptr_t)hit_region & 7) == 0 && ((uintptr_t)winners & 7) == 0 && ((uintptr_t)order & 7) == 0 &&
                ((uintptr_t)region_out & 7) == 0,
            "osb_shard_hits: misaligned hit list, winners or output");
  const size_t need = osb_shard_hits_workspace_bytes(n_hits);
  OSB_CHECK(ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 255) == 0,
            "osb_shard_hits: 256-byte aligned workspace of %zu bytes required (got %zu)", need, ws_bytes);
  uint8_t *w = reinterpret_cast<uint8_t *>(ws);
  auto take = [&](size_t bytes) { uint8_t *p = w; w += (bytes + 255) & ~size_t(255); return p; };
  uint64_t *ka = reinterpret_cast<uint64_t *>(take((size_t)n_hits * 8));
  uint64_t *kb = reinterpret_cast<uint64_t *>(take((size_t)n_hits * 8));
  int32_t *va = reinterpret_cast<int32_t *>(take((size_t)n_hits * 4));
  int32_t *vb = reinterpret_cast<int32_t *>(take((size_t)n_hits * 4));
  void *sort_ws = w;
  const int blocks = (int)ceil_div(n_hits, 256);
  k_shard_hit_keys<<<blocks, 256, 0, stream>>>(hit_query, hit_grow, n_hits, ka);
  OSB_LAUNCH_CHECK();
  // (query << 48) | global row: distinct per hit, bits 0 .. 48 + bits(nq)
  const int where = radix_sort_pairs(ka, va, kb, vb, nullptr, n_hits, 0, 48 + sh_bits_for((uint64_t)nq), sort_ws, stream);
  OSB_CHECK(where >= 0, "osb_shard_hits: sort launch failed");
  k_shard_hit_finish<<<blocks, 256, 0, stream>>>(where ? vb : va, n_hits, hit_query, hit_rank, hit_region, winners, R,
                                                 order, region_out);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
