// PTX wrappers shared by the tensor-core kernels (sm_90a): mbarrier, TMA, cp.async, wgmma.
#pragma once
#include "common.cuh"

#include <cuda.h>
#include <cudaTypedefs.h>

namespace osb {

// ------------------------------------------------------------------------------------ PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t it = 0; !done; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (it > (1u << 26)) __trap();   // a lost TMA / MMA completion must not hang the GPU
  }
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
// this thread's arrival on `bar` fires when all of its prior cp.async have landed (count pre-armed at init)
__device__ __forceinline__ void cp_async_arrive_noinc(uint32_t bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}" : "=r"(pred));
  return pred != 0;
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *tm, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(tm), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// ------------------------------------------------------------------------------------ wgmma (one warpgroup)
// D[64 x N] += A[64 x 16] B[16 x N] with both operands in shared memory and fp32 accumulators in registers.  Fragment of D:
// warp w of the warpgroup holds rows 16w + lane/4 and 16w + lane/4 + 8; of every 8-column group i it holds columns
// 8i + 2(lane%4) + {0, 1}:  d[4i + 0, 1] (first row), d[4i + 2, 3] (second row).  The N = 64 form writes the same
// registers as two N = 32 forms side by side, so accumulators are kept as 16-float blocks of 32 columns.
// TA / TB = 1: the operand is MN-major (transposed) in shared memory.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the accumulator registers must not be touched by other instructions while wgmmas on them are in flight
template <int R> __device__ __forceinline__ void wgmma_hold(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// the same forms for bf16 and fp16 operands
#define OSB_WGMMA_N32(TY) \
template <int TA, int TB> \
__device__ __forceinline__ void wgmma_n32_##TY(float *d, uint64_t da, uint64_t db, uint32_t acc) { \
  asm volatile( \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t" \
      "wgmma.mma_async.sync.aligned.m64n32k16.f32." #TY "." #TY " " \
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, %16, %17, p, 1, 1, %19, %20;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB)); \
}
OSB_WGMMA_N32(bf16)
OSB_WGMMA_N32(f16)
#undef OSB_WGMMA_N32

#define OSB_WGMMA_N64(TY) \
template <int TA, int TB> \
__device__ __forceinline__ void wgmma_n64_##TY(float *d, uint64_t da, uint64_t db, uint32_t acc) { \
  asm volatile( \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t" \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." #TY "." #TY " " \
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, %35, %36;\n\t}" \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
      : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB)); \
}
OSB_WGMMA_N64(bf16)
OSB_WGMMA_N64(f16)
#undef OSB_WGMMA_N64

// K-major, 128-byte swizzle: 8-row groups 1024 B apart (SBO); +2 advances K by 16 elements of 2 bytes
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// MN-major, 128-byte swizzle: 8 K-rows = one 1024-byte atom (SBO), 64-element MN chunks LBO bytes apart
__device__ __forceinline__ uint64_t gmma_desc_mn(uint32_t saddr, uint32_t lbo_bytes) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | (64ull << 32) | (1ull << 62);
}

// One 32-channel block of split operands (128-byte line per row: [hi ch0-15 | hi ch16-31 | lo ch0-15 | lo ch16-31]),
// both K-major: D += A_hi W_hi + A_hi W_lo + A_lo W_hi over 32 channels, N = 32 * NCH columns (B rows 4 KB per 32).
template <int NCH>
__device__ __forceinline__ void wg_split_mma(float *acc, uint64_t da, uint64_t db) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int pr = 0; pr < 3; ++pr) {
      const uint64_t a = da + 2 * h + (pr == 2 ? 4 : 0), b = db + 2 * h + (pr == 1 ? 4 : 0);
#pragma unroll
      for (int c = 0; c + 2 <= NCH; c += 2) wgmma_n64_bf16<0, 0>(acc + 16 * c, a, b + 256 * c, 1u);
      if (NCH & 1) wgmma_n32_bf16<0, 0>(acc + 16 * (NCH - 1), a, b + 256 * (NCH - 1), 1u);
    }
  }
}

// ------------------------------------------------------------------------------------ fragment epilogue
// One warp's 16 accumulator rows of one 32-column block (y[16] in the fragment order above) pass through a 2 KB staging tile
// (16 rows x 128 B, 128B swizzle), so that global loads / stores move full 128-byte lines.
__device__ __forceinline__ uint32_t stg_at(uint32_t stg, int r, int chunk) { return stg + r * 128 + ((chunk ^ (r & 7)) << 4); }

__device__ __forceinline__ void frag_stage_f32(uint32_t stg, const float *y, int lane) {   // fp32 line: 32 x 4 B
  const int r = lane >> 2, q = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(stg_at(stg, r + 8 * h, 2 * i + (q >> 1)) + 8 * (q & 1)),
                   "f"(y[4 * i + 2 * h]), "f"(y[4 * i + 2 * h + 1]) : "memory");
}
__device__ __forceinline__ void frag_stage_split(uint32_t stg, const float *y, int lane) {  // split line: hi at chunk i, lo at 4 + i
  const int r = lane >> 2, q = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      __nv_bfloat162 hi, lo;
      split_bf16(y[4 * i + 2 * h], hi.x, lo.x);
      split_bf16(y[4 * i + 2 * h + 1], hi.y, lo.y);
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg_at(stg, r + 8 * h, i) + 4 * q), "r"(*reinterpret_cast<uint32_t *>(&hi)) : "memory");
      asm volatile("st.shared.b32 [%0], %1;" ::"r"(stg_at(stg, r + 8 * h, 4 + i) + 4 * q), "r"(*reinterpret_cast<uint32_t *>(&lo)) : "memory");
    }
}
__device__ __forceinline__ void frag_add_split(uint32_t stg, float *y, int lane) {         // y += the staged split line
  const int r = lane >> 2, q = lane & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t hv, lv;
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(hv) : "r"(stg_at(stg, r + 8 * h, i) + 4 * q));
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(lv) : "r"(stg_at(stg, r + 8 * h, 4 + i) + 4 * q));
      const __nv_bfloat162 hh = *reinterpret_cast<__nv_bfloat162 *>(&hv), ll = *reinterpret_cast<__nv_bfloat162 *>(&lv);
      y[4 * i + 2 * h] += join_bf16(hh.x, ll.x);
      y[4 * i + 2 * h + 1] += join_bf16(hh.y, ll.y);
    }
}
// rows [row0, row0 + 16) of a row-major global tensor (128 bytes at col_byte of each row) -> staging; rows >= n_rows: zeros
__device__ __forceinline__ void stage_load(uint32_t stg, const uint8_t *base, int64_t row0, int64_t n_rows, int64_t row_bytes,
                                           int64_t col_byte, int lane) {
  const int chunk = lane & 7;
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int r = 4 * it + (lane >> 3);
    uint4 v = make_uint4(0, 0, 0, 0);
    if (row0 + r < n_rows) v = __ldcg(reinterpret_cast<const uint4 *>(base + (row0 + r) * row_bytes + col_byte + chunk * 16));
    asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(stg_at(stg, r, chunk)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  }
}
// staging -> global: tile row r goes to row dst_row(r) (negative: dropped)
template <class F>
__device__ __forceinline__ void stage_flush(uint32_t stg, uint8_t *base, int64_t row_bytes, int64_t col_byte, int lane, F dst_row) {
  const int chunk = lane & 7;
  uint4 v[4];
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int r = 4 * it + (lane >> 3);
    asm volatile("ld.shared.v4.b32 {%0,%1,%2,%3}, [%4];" : "=r"(v[it].x), "=r"(v[it].y), "=r"(v[it].z), "=r"(v[it].w) : "r"(stg_at(stg, r, chunk)));
  }
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int64_t g = dst_row(4 * it + (lane >> 3));
    if (g >= 0) *reinterpret_cast<uint4 *>(base + g * row_bytes + col_byte + chunk * 16) = v[it];
  }
}


// 2-D tensor map over a row-major [rows, cols_elems] tensor of 2-byte elements; box {64 elems, box_rows}; 128B swizzle
int make_tmap_2b(CUtensorMap *tm, const void *base, uint64_t cols_elems, uint64_t rows, uint32_t box_rows, int is_f16);

}  // namespace osb
