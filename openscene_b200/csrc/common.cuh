// Shared helpers for libosb200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "../../include/osb200.h"

namespace osb {

void set_error(const char *fmt, ...);
extern std::atomic<int64_t> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }

#define OSB_CHECK(cond, ...)                                                        \
  do {                                                                              \
    if (!(cond)) { ::osb::set_error(__VA_ARGS__); return 1; }                       \
  } while (0)

#define OSB_CUDA(expr)                                                              \
  do {                                                                              \
    cudaError_t _e = (expr);                                                        \
    if (_e != cudaSuccess) {                                                        \
      ::osb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return 1;                                                                     \
    }                                                                               \
  } while (0)

#define OSB_LAUNCH_CHECK()                                                          \
  do {                                                                              \
    ::osb::count_launch();                                                          \
    cudaError_t _e = cudaGetLastError();                                            \
    if (_e != cudaSuccess) {                                                        \
      ::osb::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return 1;                                                                     \
    }                                                                               \
  } while (0)

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-DEVICE property of a kernel: remember it per device (a process
// may drive several GPUs, and autograd's backward thread calls in from another host thread).  Setting it twice is harmless.
struct PerDeviceOnce {
  std::atomic<unsigned long long> done{0};
  bool need(int *dev_out) {
    int dev = 0;
    cudaGetDevice(&dev);
    *dev_out = dev;
    return dev < 0 || dev >= 64 || !((done.load(std::memory_order_acquire) >> dev) & 1ull);
  }
  void mark(int dev) { if (dev >= 0 && dev < 64) done.fetch_or(1ull << dev, std::memory_order_release); }
};
#define OSB_SMEM_ATTR_ONCE(kernel, bytes)                                                              \
  do {                                                                                                 \
    static ::osb::PerDeviceOnce _once;                                                                 \
    int _dev;                                                                                          \
    if (_once.need(&_dev)) {                                                                           \
      OSB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))); \
      _once.mark(_dev);                                                                                \
    }                                                                                                  \
  } while (0)

// ---------------------------------------------------------------------------------------------
// Coordinate keys.  Fields: x,y,z biased by 2^17 into 18 bits each, batch in the top 10 bits.
//   pack   = b<<54 | z<<36 | y<<18 | x        (hash key; neighbour = one 64-bit add)
//   morton = b<<54 | interleave(x,y,z)        (sort key; x is the least significant of each triple)
// ---------------------------------------------------------------------------------------------
constexpr int      kCoordBias  = 1 << 17;
constexpr int      kCoordLimit = (1 << 17) - 256;
constexpr uint64_t kEmptyKey   = 0xFFFFFFFFFFFFFFFFull;

struct __align__(16) HashSlot {
  unsigned long long key;
  int32_t            row;
  int32_t            pad;
};

__host__ __device__ inline uint64_t pack_key(int b, int x, int y, int z) {
  return ((uint64_t)(uint32_t)b << 54) | ((uint64_t)(uint32_t)(z + kCoordBias) << 36) |
         ((uint64_t)(uint32_t)(y + kCoordBias) << 18) | (uint64_t)(uint32_t)(x + kCoordBias);
}
// signed per-axis delta as one 64-bit addend (fields never borrow inside the valid range)
__host__ __device__ inline uint64_t pack_delta(int dx, int dy, int dz) {
  return (uint64_t)((int64_t)dx + ((int64_t)dy << 18) + ((int64_t)dz << 36));
}
__host__ __device__ inline uint64_t spread3(uint32_t v) {  // 18 bits -> every third bit
  uint64_t x = v & 0x3FFFFu;
  x = (x | (x << 32)) & 0x001F00000000FFFFull;
  x = (x | (x << 16)) & 0x001F0000FF0000FFull;
  x = (x | (x << 8)) & 0x100F00F00F00F00Full;
  x = (x | (x << 4)) & 0x10C30C30C30C30C3ull;
  x = (x | (x << 2)) & 0x1249249249249249ull;
  return x;
}
__host__ __device__ inline uint64_t morton_key(int b, int x, int y, int z) {
  return ((uint64_t)(uint32_t)b << 54) | spread3((uint32_t)(x + kCoordBias)) |
         (spread3((uint32_t)(y + kCoordBias)) << 1) | (spread3((uint32_t)(z + kCoordBias)) << 2);
}
__host__ __device__ inline uint64_t hash_u64(uint64_t k) {
  k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
  return k;
}

__device__ inline int hash_lookup(const HashSlot *__restrict__ slots, uint64_t mask, uint64_t key) {
  uint64_t s = hash_u64(key) & mask;
  while (true) {
    // 16-byte slot read in one transaction
    const int4 v = __ldg(reinterpret_cast<const int4 *>(slots + s));
    const uint64_t k = ((uint64_t)(uint32_t)v.y << 32) | (uint32_t)v.x;
    if (k == key) return v.z;
    if (k == kEmptyKey) return -1;
    s = (s + 1) & mask;
  }
}

// ---------------------------------------------------------------------------------------------
// Occupancy grid: the alternative to the hash for coordinate sets that are non-negative and fit 2^27 cells
// (every indoor scene; the coarse levels of lidar sweeps).  One bit per cell of a 2^nbits cube per batch index, cells in
// Morton order (x least significant), so a 64-bit word is one aligned 4x4x4 block.  Rows of a coordinate set are
// Morton sorted, hence the rows of a word are contiguous and
//        row(cell) = first_row[word] + popc(bits of the word below the cell).
// A lookup is two loads from a table of a few MB that neighbouring voxels share (L1 / L2 resident) instead of a probe
// chain of 16-byte slots scattered over a table 4x the set.
// ---------------------------------------------------------------------------------------------
struct OccGridView {
  const unsigned long long *bitmap;   // [n_batch * words_per_batch]
  const int32_t *first_row;           // [n_batch * words_per_batch], defined where bitmap != 0
  int nbits;                          // cells per axis = 1 << nbits (2 <= nbits <= 9)
  int log2_ts;                        // cell = coordinate >> log2_ts (coordinates of the set are multiples of the tensor stride)
  int n_batch;
};
__host__ __device__ inline uint32_t spread3_10(uint32_t x) {   // 10 bits -> every third bit of 30
  x &= 0x3FFu;
  x = (x | (x << 16)) & 0x030000FFu;
  x = (x | (x << 8)) & 0x0300F00Fu;
  x = (x | (x << 4)) & 0x030C30C3u;
  x = (x | (x << 2)) & 0x09249249u;
  return x;
}
__host__ __device__ inline int64_t occgrid_words_per_batch(int nbits) { return (int64_t)1 << (3 * nbits - 6); }
// (word, bit) of a coordinate that is known to lie inside the grid
__device__ inline void occgrid_cell(const OccGridView &g, int b, int x, int y, int z, int64_t &word, int &bit) {
  const uint32_t m = spread3_10((uint32_t)(x >> g.log2_ts)) | (spread3_10((uint32_t)(y >> g.log2_ts)) << 1) |
                     (spread3_10((uint32_t)(z >> g.log2_ts)) << 2);
  word = (int64_t)b * occgrid_words_per_batch(g.nbits) + (m >> 6);
  bit = (int)(m & 63u);
}
__device__ inline int occgrid_lookup(const OccGridView &g, int b, int x, int y, int z) {
  const uint32_t lim = 1u << g.nbits;
  const int ts_mask = (1 << g.log2_ts) - 1;
  // arithmetic shifts keep negatives negative -> they fail the unsigned bound test; off-lattice queries cannot match
  if ((uint32_t)(x >> g.log2_ts) >= lim || (uint32_t)(y >> g.log2_ts) >= lim || (uint32_t)(z >> g.log2_ts) >= lim ||
      (uint32_t)b >= (uint32_t)g.n_batch || ((x | y | z) & ts_mask))
    return -1;
  int64_t word; int bit;
  occgrid_cell(g, b, x, y, z, word, bit);
  const unsigned long long w = __ldg(g.bitmap + word);
  if (!((w >> bit) & 1ull)) return -1;
  return __ldg(g.first_row + word) + __popcll(w & ((1ull << bit) - 1ull));
}

// ---------------------------------------------------------------------------------------------
// split-fp32: v ~= hi + lo, both bf16 (round-to-nearest-even).  |v - hi - lo| <= 2^-17 |v|.
// ---------------------------------------------------------------------------------------------
__device__ inline void split_bf16(float v, __nv_bfloat16 &hi, __nv_bfloat16 &lo) {
  hi = __float2bfloat16_rn(v);
  lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
__device__ inline float join_bf16(__nv_bfloat16 hi, __nv_bfloat16 lo) {
  return __bfloat162float(hi) + __bfloat162float(lo);
}
// byte offset of channel c (hi part) inside a split row; the lo part is +64 bytes
__host__ __device__ inline int split_off_hi(int c) { return (c >> 5) * 128 + (c & 31) * 2; }

// The split-bf16 B operand of the tensor-core convolutions (osb_conv_pack_weights, osb_conv_repack): K * cout_pad rows, row
// kn = k * cout_pad + n holding input channels 0..cin-1 of output column n as split lines; rows n >= cout are zero.
// Writes packed element e (channel e % cin of row e / cin); weight element (k, n, c) is read at w[k * sk + n * sn + c * sc].
__device__ inline void pack_weight_elem(const float *__restrict__ w, int64_t sk, int64_t sn, int64_t sc, int cin, int cout,
                                        int cout_pad, int64_t e, uint8_t *__restrict__ wpack) {
  const int c = (int)(e % cin);
  const int64_t kn = e / cin;
  const int n = (int)(kn % cout_pad), k = (int)(kn / cout_pad);
  float v = 0.f;
  if (n < cout) v = w[k * sk + n * sn + c * sc];
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  uint8_t *row = wpack + kn * (int64_t)cin * 4 + split_off_hi(c);
  *reinterpret_cast<__nv_bfloat16 *>(row) = hi;
  *reinterpret_cast<__nv_bfloat16 *>(row + 64) = lo;
}

}  // namespace osb
