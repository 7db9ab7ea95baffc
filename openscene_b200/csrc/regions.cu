// Regions of search hits (DESIGN.md, "Region contract"): the hits of each (scene, query), as osb_search_hits lists them in
// (query, global row) order, grouped into connected components under Chebyshev distance <= reach on their voxel
// coordinates, and the R best components per query.
//
//   k_rg_init      gather each hit's coordinates (one 16-byte load), pack them into 18 bits per axis, range check
//   sort 1 / 2     stable radix sort by packed coordinate, then stable by (query, scene) segment: each segment occupies the
//                  same positions as in the hit list, its hits now in coordinate order
//   k_rg_link      per hit and per (dx, dy) of the positive half of the offsets: binary search of the first key at dz = -reach
//                  inside its own segment, then a scan up to dz = +reach; each neighbour pair is linked once.  Union by
//                  index: the larger root is hooked under the smaller with atomicCAS, so a component's root is its
//                  smallest hit index (its smallest global row) whatever order threads arrive in
//   k_rg_compress  full path compression
//   k_rg_stats     per root: size (atomicAdd), box (atomicMin / atomicMax per axis), best hit (64-bit atomicMax of its
//                  search key)
//   sort 3         roots with size >= min_voxels by (query, descending best key); everything else sorts last
//   k_rg_finish    the first R of each query decoded; k_rg_hits the optional per-hit outputs
// Integer atomics only, and every result is a function of the partition, which is unique: two calls give the same bits.
#include "match_tc.cuh"
#include "sortscan.cuh"
#include <algorithm>
#include <climits>

namespace osb {

constexpr int RG_BIAS = 1 << 17;                 // coordinate + 2^17 fits 18 bits inside the coordinate-set range
constexpr int RG_LIMIT = (1 << 17) - 256;        // |x|, |y|, |z| < 2^17 - 256, as osb_coordset_build
constexpr uint64_t RG_INVALID = ~0ull;

__device__ __forceinline__ uint64_t rg_pack(int x, int y, int z) {
  return ((uint64_t)(x + RG_BIAS) << 36) | ((uint64_t)(y + RG_BIAS) << 18) | (uint64_t)(z + RG_BIAS);
}
__device__ __forceinline__ int rg_axis(uint64_t p, int a) {
  return (int)((p >> (36 - 18 * a)) & 0x3ffffu) - RG_BIAS;
}

struct RegionWs {
  uint64_t *pc;          // [H] packed coordinate of hit i
  uint64_t *ka, *kb;     // [H] sort keys
  int32_t *va, *vb;      // [H] sort payloads
  int32_t *parent;       // [H]
  uint32_t *size;        // [H] per root
  int32_t *bmin, *bmax;  // [3][H] per root
  unsigned long long *best;   // [H] per root
  int32_t *rank_of;      // [H] per root: rank in its query's list or -1
  void *sort_ws;
};

static size_t rg_carve(int64_t H, uint8_t *w, RegionWs *r) {
  uint8_t *const w0 = w;
  auto take = [&](size_t bytes) { uint8_t *p = w; w += (bytes + 255) & ~size_t(255); return p; };
  const size_t n = (size_t)H;
  r->pc = reinterpret_cast<uint64_t *>(take(n * 8));
  r->ka = reinterpret_cast<uint64_t *>(take(n * 8));
  r->kb = reinterpret_cast<uint64_t *>(take(n * 8));
  r->best = reinterpret_cast<unsigned long long *>(take(n * 8));
  r->va = reinterpret_cast<int32_t *>(take(n * 4));
  r->vb = reinterpret_cast<int32_t *>(take(n * 4));
  r->parent = reinterpret_cast<int32_t *>(take(n * 4));
  r->size = reinterpret_cast<uint32_t *>(take(n * 4));
  r->rank_of = reinterpret_cast<int32_t *>(take(n * 4));
  r->bmin = reinterpret_cast<int32_t *>(take(n * 12));
  r->bmax = reinterpret_cast<int32_t *>(take(n * 12));
  r->sort_ws = take(radix_sort_ws_bytes(H));
  return (size_t)(w - w0);
}

__global__ void k_rg_init(const int64_t *__restrict__ hit_key, int64_t H, const int4 *__restrict__ coords, int64_t n_rows,
                          int nq, RegionWs r, int *status) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H) return;
  const uint64_t key = (uint64_t)hit_key[i];
  int64_t g = (int64_t)(key & 0xffffffffu);
  if ((int64_t)(key >> 32) >= nq || g >= n_rows) { atomicOr(status, OSB_REGIONS_ST_COUNT); g = 0; }
  const int4 c = __ldg(coords + g);
  int x = c.x, y = c.y, z = c.z;
  if (abs(x) >= RG_LIMIT || abs(y) >= RG_LIMIT || abs(z) >= RG_LIMIT || x == INT_MIN || y == INT_MIN || z == INT_MIN) {
    atomicOr(status, OSB_REGIONS_ST_RANGE);
    x = y = z = 0;
  }
  const uint64_t p = rg_pack(x, y, z);
  r.pc[i] = p;
  r.ka[i] = p;
  r.parent[i] = (int32_t)i;
  r.size[i] = 0;
  r.best[i] = 0;
#pragma unroll
  for (int a = 0; a < 3; ++a) { r.bmin[a * H + i] = INT_MAX; r.bmax[a * H + i] = INT_MIN; }
}

// segment (query * S + scene) of the hit at sorted position j
__global__ void k_rg_segkey(const int64_t *__restrict__ hit_key, const int32_t *__restrict__ perm, int64_t H,
                            const int32_t *__restrict__ row_scene, int64_t n_rows, int64_t n_scenes, uint64_t *seg) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= H) return;
  const uint64_t key = (uint64_t)hit_key[perm[j]];
  const int64_t g = std::min<int64_t>((int64_t)(key & 0xffffffffu), n_rows - 1);
  seg[j] = (key >> 32) * (uint64_t)n_scenes + (uint64_t)__ldg(row_scene + g);
}

__global__ void k_rg_gather_pc(const uint64_t *__restrict__ pc, const int32_t *__restrict__ perm, int64_t H, uint64_t *spc) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < H) spc[j] = pc[perm[j]];
}

__device__ __forceinline__ int rg_find(int32_t *parent, int x) {
  volatile int32_t *P = parent;
  int p = P[x];
  while (p != x) {
    const int gp = P[p];
    if (gp != p) P[x] = gp;           // path halving: gp is an ancestor of x, whatever other threads write meanwhile
    x = p;
    p = gp;
  }
  return x;
}

__device__ __forceinline__ void rg_unite(int32_t *parent, int a, int b) {
  for (;;) {
    a = rg_find(parent, a);
    b = rg_find(parent, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicCAS(parent + b, b, a);   // hook the larger root under the smaller
    if (old == b) return;
  }
}

// first position in [lo, hi) whose key is >= v
__device__ __forceinline__ int64_t rg_lower(const uint64_t *__restrict__ k, int64_t lo, int64_t hi, uint64_t v) {
  while (lo < hi) {
    const int64_t m = (lo + hi) >> 1;
    if (k[m] < v) lo = m + 1; else hi = m;
  }
  return lo;
}

__global__ void k_rg_link(const uint64_t *__restrict__ spc, const uint64_t *__restrict__ seg, const int32_t *__restrict__ perm,
                          int64_t H, int reach, int32_t *parent, int *status) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= H) return;
  const uint64_t sg = seg[j], v = spc[j];
  const int64_t hi = rg_lower(seg, j + 1, H, sg + 1);      // end of the segment; every positive offset lies above v
  const int self = perm[j];
  if (j + 1 < hi && spc[j + 1] == v) atomicOr(status, OSB_REGIONS_ST_DUP);
  for (int64_t t = j + 1; t < hi && spc[t] <= v + (uint64_t)reach; ++t)       // (0, 0, 1 .. reach)
    if (spc[t] != v) rg_unite(parent, self, perm[t]);
  for (int dx = 0; dx <= reach; ++dx)
    for (int dy = dx ? -reach : 1; dy <= reach; ++dy) {
      const uint64_t c = v + ((int64_t)dx << 36) + ((int64_t)dy << 18);
      const uint64_t a = c - (uint64_t)reach, b = c + (uint64_t)reach;
      for (int64_t t = rg_lower(spc, j + 1, hi, a); t < hi && spc[t] <= b; ++t) rg_unite(parent, self, perm[t]);
    }
}

// full path compression once every link is made: a read-only walk, so that no thread overwrites a root another thread
// has already stored
__global__ void k_rg_compress(int32_t *parent, int64_t H) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H) return;
  volatile int32_t *P = parent;
  int x = (int)i, p = P[x];
  while (p != x) { x = p; p = P[x]; }
  P[i] = x;
}

__global__ void k_rg_stats(const int64_t *__restrict__ hit_key, const __half *__restrict__ hit_score, int64_t H, RegionWs r) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H) return;
  const int root = r.parent[i];
  const uint64_t p = r.pc[i];
  atomicAdd(r.size + root, 1u);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    atomicMin(r.bmin + a * H + root, rg_axis(p, a));
    atomicMax(r.bmax + a * H + root, rg_axis(p, a));
  }
  atomicMax(r.best + root, (unsigned long long)search_key(hit_score[i], (int64_t)((uint64_t)hit_key[i] & 0xffffffffu)));
}

// sort key of every hit: roots with size >= min_voxels by (query, descending best key), the rest last
__global__ void k_rg_rank_keys(const int64_t *__restrict__ hit_key, int64_t H, const int32_t *__restrict__ row_scene,
                               int64_t n_rows, int nq, int min_voxels, RegionWs r, unsigned long long *n_regions) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H) return;
  r.rank_of[i] = -1;
  uint64_t key = RG_INVALID;
  if (r.parent[i] == (int32_t)i && r.size[i] >= (uint32_t)min_voxels) {
    const uint64_t hk = (uint64_t)hit_key[i], q = hk >> 32;
    const int64_t g = std::min<int64_t>((int64_t)(hk & 0xffffffffu), n_rows - 1);
    key = (q << 48) | (~(r.best[i] >> 16) & 0xffffffffffffull);
    atomicAdd(n_regions + (size_t)__ldg(row_scene + g) * nq + q, 1ull);
  }
  r.ka[i] = key;
}

// block q: the first R keys of query q
__global__ void k_rg_finish(const uint64_t *__restrict__ keys, const int32_t *__restrict__ idx, int64_t H, int R, RegionWs r,
                            const int32_t *__restrict__ row_scene, const int64_t *__restrict__ scene_off, __half *score,
                            int64_t *scene, int64_t *row, int64_t *size, int32_t *box_min, int32_t *box_max) {
  const int q = blockIdx.x, t = threadIdx.x;
  if (t >= R) return;
  const int64_t start = H ? rg_lower(keys, 0, H, (uint64_t)q << 48) : 0, j = start + t;
  const size_t o = (size_t)q * R + t;
  if (j < H && (keys[j] >> 48) == (uint64_t)q) {
    const int i = idx[j];
    const unsigned long long b = r.best[i];
    const int64_t g = (int64_t)(~(uint32_t)(b >> 16));
    const int s = row_scene[g];
    score[o] = __ushort_as_half((unsigned short)(b & 0xffffu));
    scene[o] = s;
    row[o] = g - scene_off[s];
    size[o] = r.size[i];
#pragma unroll
    for (int a = 0; a < 3; ++a) { box_min[3 * o + a] = r.bmin[a * H + i]; box_max[3 * o + a] = r.bmax[a * H + i]; }
    r.rank_of[i] = t;
  } else {
    score[o] = __ushort_as_half((unsigned short)0xfc00u);
    scene[o] = -1;
    row[o] = -1;
    size[o] = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) { box_min[3 * o + a] = 0; box_max[3 * o + a] = 0; }
  }
}

__global__ void k_rg_hits(const int64_t *__restrict__ hit_key, int64_t H, const int32_t *__restrict__ row_scene,
                          const int64_t *__restrict__ scene_off, int64_t n_rows, RegionWs r, int64_t *hit_query,
                          int64_t *hit_scene, int64_t *hit_row, int64_t *hit_region) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= H) return;
  const uint64_t hk = (uint64_t)hit_key[i];
  const int64_t g = std::min<int64_t>((int64_t)(hk & 0xffffffffu), n_rows - 1);
  const int s = row_scene[g];
  hit_query[i] = (int64_t)(hk >> 32);
  hit_scene[i] = s;
  hit_row[i] = g - scene_off[s];
  hit_region[i] = r.rank_of[r.parent[i]];
}

static inline int bits_for(uint64_t n) {   // bits of the largest value below n
  int b = 0;
  while (b < 64 && (n - 1) >> b) ++b;
  return b;
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_regions_workspace_bytes(int64_t n_hits) {
  if (n_hits < 0 || n_hits >= (int64_t(1) << 31)) return 0;
  RegionWs r;
  return rg_carve(n_hits, nullptr, &r);
}

int osb_regions(const int64_t *hit_key, const void *hit_score_f16, int64_t n_hits, const int32_t *coords,
                const int32_t *row_scene, const int64_t *scene_off, int64_t n_rows, int64_t n_scenes, int32_t nq, int32_t R,
                int32_t reach, int32_t min_voxels, void *score_f16, int64_t *scene, int64_t *row, int64_t *size,
                int32_t *box_min, int32_t *box_max, int64_t *n_regions, int64_t *hit_query, int64_t *hit_scene,
                int64_t *hit_row, int64_t *hit_region, int32_t *status, void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(nq >= 1 && nq <= OSB_SEARCH_MAX_QUERIES, "osb_regions: nq=%d outside 1..%d", nq, OSB_SEARCH_MAX_QUERIES);
  OSB_CHECK(R >= 1 && R <= OSB_REGIONS_MAX_R, "osb_regions: R=%d outside 1..%d", R, OSB_REGIONS_MAX_R);
  OSB_CHECK(reach >= 1 && reach <= 2, "osb_regions: reach=%d outside 1..2", reach);
  OSB_CHECK(min_voxels >= 1, "osb_regions: min_voxels=%d below 1", min_voxels);
  OSB_CHECK(n_rows >= 1 && n_rows < (int64_t(1) << 31), "osb_regions: N=%lld outside 1..2^31-1", (long long)n_rows);
  OSB_CHECK(n_scenes >= 1 && n_scenes <= n_rows, "osb_regions: %lld scenes for %lld rows", (long long)n_scenes,
            (long long)n_rows);
  OSB_CHECK(n_hits >= 0 && n_hits < (int64_t(1) << 31), "osb_regions: n_hits=%lld outside 0..2^31-1", (long long)n_hits);
  OSB_CHECK(coords && row_scene && scene_off && status, "osb_regions: NULL coordinates, row scenes, scene offsets or status");
  OSB_CHECK(n_hits == 0 || (hit_key && hit_score_f16), "osb_regions: NULL hit list");
  OSB_CHECK(score_f16 && scene && row && size && box_min && box_max && n_regions, "osb_regions: NULL region output");
  const bool hits = hit_query != nullptr;
  OSB_CHECK(hits == (hit_scene != nullptr) && hits == (hit_row != nullptr) && hits == (hit_region != nullptr),
            "osb_regions: hit_query, hit_scene, hit_row and hit_region go together");
  OSB_CHECK(((uintptr_t)coords & 15) == 0, "osb_regions: coordinates must be 16-byte aligned");
  OSB_CHECK(((uintptr_t)hit_key & 7) == 0 && ((uintptr_t)hit_score_f16 & 1) == 0 && ((uintptr_t)status & 3) == 0,
            "osb_regions: misaligned hit list or status");
  const size_t need = osb_regions_workspace_bytes(n_hits);
  OSB_CHECK(n_hits == 0 || (ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 255) == 0),
            "osb_regions: 256-byte aligned workspace of %zu bytes required (got %zu)", need, ws_bytes);

  OSB_CUDA(cudaMemsetAsync(n_regions, 0, (size_t)n_scenes * nq * 8, stream));
  RegionWs r{};
  const int64_t H = n_hits;
  if (H > 0) {
    rg_carve(H, reinterpret_cast<uint8_t *>(ws), &r);
    const int blocks = (int)ceil_div(H, 256);
    k_rg_init<<<blocks, 256, 0, stream>>>(hit_key, H, reinterpret_cast<const int4 *>(coords), n_rows, nq, r, status);
    OSB_LAUNCH_CHECK();
    // sort 1: packed coordinate (54 bits), payload = hit index
    int w = radix_sort_pairs(r.ka, r.va, r.kb, r.vb, nullptr, H, 0, 54, r.sort_ws, stream);
    OSB_CHECK(w >= 0, "osb_regions: sort launch failed");
    uint64_t *k1 = w ? r.kb : r.ka, *k2 = w ? r.ka : r.kb;
    int32_t *p1 = w ? r.vb : r.va, *p2 = w ? r.va : r.vb;
    // sort 2: stable by (query, scene) segment
    k_rg_segkey<<<blocks, 256, 0, stream>>>(hit_key, p1, H, row_scene, n_rows, n_scenes, k2);
    OSB_LAUNCH_CHECK();
    w = radix_sort_pairs(k2, p1, k1, p2, p1, H, 0, bits_for((uint64_t)nq * n_scenes), r.sort_ws, stream);
    OSB_CHECK(w >= 0, "osb_regions: sort launch failed");
    uint64_t *seg = w ? k1 : k2, *spc = w ? k2 : k1;
    const int32_t *perm = w ? p2 : p1;
    k_rg_gather_pc<<<blocks, 256, 0, stream>>>(r.pc, perm, H, spc);
    OSB_LAUNCH_CHECK();
    k_rg_link<<<blocks, 256, 0, stream>>>(spc, seg, perm, H, reach, r.parent, status);
    OSB_LAUNCH_CHECK();
    k_rg_compress<<<blocks, 256, 0, stream>>>(r.parent, H);
    OSB_LAUNCH_CHECK();
    k_rg_stats<<<blocks, 256, 0, stream>>>(hit_key, (const __half *)hit_score_f16, H, r);
    OSB_LAUNCH_CHECK();
    k_rg_rank_keys<<<blocks, 256, 0, stream>>>(hit_key, H, row_scene, n_rows, nq, min_voxels, r,
                                               reinterpret_cast<unsigned long long *>(n_regions));
    OSB_LAUNCH_CHECK();
    // sort 3: (query << 48) | ~best key (55 bits), everything else ~0 and last
    w = radix_sort_pairs(r.ka, r.va, r.kb, r.vb, nullptr, H, 0, 55, r.sort_ws, stream);
    OSB_CHECK(w >= 0, "osb_regions: sort launch failed");
    k_rg_finish<<<nq, 32, 0, stream>>>(w ? r.kb : r.ka, w ? r.vb : r.va, H, R, r, row_scene, scene_off,
                                       (__half *)score_f16, scene, row, size, box_min, box_max);
    OSB_LAUNCH_CHECK();
    if (hits) {
      k_rg_hits<<<blocks, 256, 0, stream>>>(hit_key, H, row_scene, scene_off, n_rows, r, hit_query, hit_scene, hit_row,
                                            hit_region);
      OSB_LAUNCH_CHECK();
    }
  } else {
    k_rg_finish<<<nq, 32, 0, stream>>>(nullptr, nullptr, 0, R, r, row_scene, scene_off, (__half *)score_f16, scene, row,
                                       size, box_min, box_max);
    OSB_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
