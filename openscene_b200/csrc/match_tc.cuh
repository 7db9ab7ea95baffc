// The pieces of the tensor-core match (match_tc.cu) that the scene search (search.cu) multiplies with as well: the A
// producers that load a 128-row tile and round it to the fp16 operand (mt_fill_a8: from the FP8 index's codes), the TMA
// stream of the 96-row text chunks, the wgmma pass over one 96-column block, and the 64-bit order keys.  Whatever kernel
// calls them, a score is the same fp16 rounding of the same fp32 sum in the same order.  match_tc_body calls mt_fill_a; it
// keeps its TMA and wgmma loops written out (the statements of mt_text_stage and mt_mma_pass), because calling the helpers
// there moves the register allocation of some of its instantiations, and its kernels compile to the same instructions as
// before this header existed.
#pragma once
#include <cuda_fp8.h>
#include "tc_ptx.cuh"

namespace osb {

constexpr int MT_M = 128;
constexpr int MT_NW = 96;            // text rows per MMA pass (N of the instruction)
constexpr int MT_PW = 16;             // A-producer warps (8 rows each)
constexpr int MT_THREADS = (MT_PW + 1) * 32;   // + TMA warp
constexpr int MT_BSTAGES = 2;

struct MatchTcParams {
  const void *feat;                  // [n_vox, C] fp32 or fp16
  const __half *feat2;               // optional second source (fp16) for the ensemble select
  const float *sel_a, *sel_b;        // ensemble: use feat2 where sel_a[p] < sel_b[p]
  const int64_t *inds_reverse;       // [n_pts] or NULL
  int64_t n_pts;
  int C, k_text, n_pass;
  int feat_is_f16, normalize;
  __half *scores;                    // [n_pts, k_text] or NULL
  int64_t *label;                    // [n_pts] or NULL
  float *smax;                       // [n_pts] or NULL
  __half *feat_out;                  // [n_pts, C] or NULL: the fp16 operand actually multiplied (ensemble feature)
};

// order key of score h at column k: larger is better.  Bits 48-63 map the score to an unsigned order (NaN highest, -0 as
// +0), bits 16-47 hold ~k (the lower column wins a tie), bits 0-15 the score's own fp16 bits.  Every valid key is > 0.
__device__ __forceinline__ uint64_t topk_key(__half h, int k) {
  const uint32_t b = __half_as_ushort(h);
  const uint32_t u = (b & 0x7fffu) > 0x7c00u ? 0xffffu : b == 0x8000u ? 0x8000u : (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
  return ((uint64_t)u << 48) | ((uint64_t)(~(uint32_t)k) << 16) | b;
}

// order key of the scene search (search.cu, regions.cu): bits 48-63 the score's order (-0 as +0), bits 16-47 ~row (the
// lower global row wins a tie), bits 0-15 the score's fp16 bits; NaN has key 0, below every other key.
__device__ __forceinline__ uint64_t search_key(__half h, int64_t row) {
  const uint32_t b = __half_as_ushort(h);
  if ((b & 0x7fffu) > 0x7c00u) return 0;
  const uint32_t u = b == 0x8000u ? 0x8000u : (b & 0x8000u) ? (~b & 0xffffu) : (b | 0x8000u);
  return ((uint64_t)u << 48) | ((uint64_t)(~(uint32_t)row) << 16) | b;
}

// insert key into the descending list L[0..n) unless it is below L[n-1] (keys are distinct: one per column)
__device__ __forceinline__ void topk_insert(uint64_t *L, int n, uint64_t key) {
  if (key < L[n - 1]) return;
  int j = n - 1;
  for (; j > 0 && L[j - 1] < key; --j) L[j] = L[j - 1];
  L[j] = key;
}

// A producers (warps 0..MT_PW-1): rows row0 .. row0 + 127 of the operand into the K-major 128B-swizzled tile sA of all C/64
// depth chunks, rounded to fp16 where the reference rounds.  Rows at or past n_pts are zero.  The caller fences the
// generic-proxy writes before a wgmma reads them.
template <int NP>   // half2 pairs per lane: C = 64 * NP
__device__ __forceinline__ void mt_fill_a(const MatchTcParams &p, uint8_t *sA, int64_t row0, int warp, int lane) {
  constexpr int C = 64 * NP;
  // RB rows are in flight per warp (their loads are issued before any is consumed): 16 warps x RB x 3 KB of
  // outstanding loads per SM keeps HBM busy from the single resident CTA; 16 warps also spread the
  // convert / normalise instruction stream over all four schedulers.
  constexpr int RB = 2, ROWS_PW = MT_M / MT_PW;
  for (int rr0 = 0; rr0 < ROWS_PW; rr0 += RB) {
    float v[RB][2 * NP];
    bool f16[RB], live[RB];
    float ss[RB];
#pragma unroll
    for (int u = 0; u < RB; ++u) {
      const int64_t pt = row0 + warp * ROWS_PW + rr0 + u;
      live[u] = pt < p.n_pts;
      f16[u] = false;
      ss[u] = 0.f;
      if (live[u]) {
        const int64_t vox = p.inds_reverse ? __ldg(p.inds_reverse + pt) : pt;
        bool second = false;
        if (p.feat2 != nullptr) second = (p.sel_a == nullptr) ? true : (__ldg(p.sel_a + pt) < __ldg(p.sel_b + pt));
        f16[u] = second || p.feat_is_f16;
        const void *src = second ? (const void *)p.feat2 : p.feat;
        if (f16[u]) {
          const __half2 *q = reinterpret_cast<const __half2 *>(src) + vox * (C / 2);
#pragma unroll
          for (int j = 0; j < NP; ++j) {
            const float2 f = __half22float2(__ldg(q + lane + 32 * j));
            v[u][2 * j] = f.x; v[u][2 * j + 1] = f.y;
          }
        } else {
          const float2 *q = reinterpret_cast<const float2 *>(src) + vox * (C / 2);
#pragma unroll
          for (int j = 0; j < NP; ++j) {
            const float2 f = __ldg(q + lane + 32 * j);
            v[u][2 * j] = f.x; v[u][2 * j + 1] = f.y;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 2 * NP; ++j) v[u][j] = 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < RB; ++u) {
      const int r = warp * ROWS_PW + rr0 + u;
      const int64_t pt = row0 + r;
      if (p.normalize) {
#pragma unroll
        for (int j = 0; j < 2 * NP; ++j) ss[u] = fmaf(v[u][j], v[u][j], ss[u]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss[u] += __shfl_xor_sync(0xffffffffu, ss[u], o);
        float nrm = sqrtf(ss[u]);
        float d;
        if (f16[u]) {   // the reference takes norm, +1e-5 and the division on an fp16 tensor (evaluate.py:303-305)
          nrm = __half2float(__float2half_rn(nrm));
          d = __half2float(__float2half_rn(nrm + 1e-5f));
        } else {
          d = nrm + 1e-5f;
        }
        // x / d evaluated as x * (1/d) (one rounding more than the reference's division; the following fp16
        // rounding absorbs it except for values within 2^-24 of an fp16 rounding boundary)
        const float rd = __frcp_rn(d);
#pragma unroll
        for (int j = 0; j < 2 * NP; ++j) v[u][j] = v[u][j] * rd;
      }
      // chunk j of this row: lane holds elements 2*lane, 2*lane+1 -> bytes [4*lane, 4*lane+4) of the 128-byte line
      const uint32_t line = smem_u32(sA) + r * 128 + ((((4 * lane) >> 4) ^ (r & 7)) << 4) + ((4 * lane) & 15);
#pragma unroll
      for (int j = 0; j < NP; ++j) {
        const __half2 h = __floats2half2_rn(v[u][2 * j], v[u][2 * j + 1]);       // the reference's `.half()`
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(line + j * (MT_M * 128)), "r"(*reinterpret_cast<const uint32_t *>(&h)) : "memory");
        if (p.feat_out != nullptr && live[u])
          reinterpret_cast<__half2 *>(p.feat_out)[pt * (C / 2) + lane + 32 * j] = h;
      }
    }
  }
}

// FP8 A producer (warps 0..MT_PW-1; DESIGN.md, "FP8 index contract"): rows row0 .. row0 + 127 of e4m3 codes [n, C] and
// their int8 exponents into the same K-major 128B-swizzled fp16 tile that mt_fill_a writes for the rows d = code * 2^e.
// Every d is an fp16 number (the exponent rule keeps it in range, subnormals included), and both the unpack and the fp32
// multiply by 2^e are exact, so the tile holds d bit for bit.  Rows at or past n are zero.  A lane loads 8 codes at once and
// stores their 8 halves as one 16-byte swizzled unit.
template <int NP>   // C = 64 * NP
__device__ __forceinline__ void mt_fill_a8(const uint8_t *codes, const int8_t *row_exp, int64_t n, uint8_t *sA,
                                           int64_t row0, int warp, int lane) {
  constexpr int C = 64 * NP, U = NP / 4;          // C / 8 units of 8 codes per row, U per lane
  constexpr int RB = 4, ROWS_PW = MT_M / MT_PW;    // 4 rows in flight per warp: as many bytes as mt_fill_a's 2 fp16 rows
  for (int rr0 = 0; rr0 < ROWS_PW; rr0 += RB) {
    uint2 v[RB][U];
    int e[RB];
#pragma unroll
    for (int u = 0; u < RB; ++u) {
      const int64_t pt = row0 + warp * ROWS_PW + rr0 + u;
      if (pt < n) {
        const uint2 *q = reinterpret_cast<const uint2 *>(codes + pt * C);
#pragma unroll
        for (int i = 0; i < U; ++i) v[u][i] = __ldg(q + lane + 32 * i);
        e[u] = __ldg(row_exp + pt);
      } else {
#pragma unroll
        for (int i = 0; i < U; ++i) v[u][i] = make_uint2(0u, 0u);
        e[u] = 0;
      }
    }
#pragma unroll
    for (int u = 0; u < RB; ++u) {
      const int r = warp * ROWS_PW + rr0 + u;
      const float sc = __int_as_float((127 + e[u]) << 23);                   // 2^e, e in [-15, 7]
#pragma unroll
      for (int i = 0; i < U; ++i) {
        const int w = lane + 32 * i;   // elements 8w .. 8w + 7: depth chunk w / 8, 16-byte unit w % 8 of the 128-byte line
        uint32_t h[4];
#pragma unroll
        for (int p = 0; p < 4; ++p) {
          const uint32_t word = p < 2 ? v[u][i].x : v[u][i].y;
          const __half2_raw raw = __nv_cvt_fp8x2_to_halfraw2((__nv_fp8x2_storage_t)(word >> (16 * (p & 1))), __NV_E4M3);
          const float2 f = __half22float2(__half2(raw));
          const __half2 d = __floats2half2_rn(f.x * sc, f.y * sc);
          h[p] = *reinterpret_cast<const uint32_t *>(&d);
        }
        const uint32_t addr = smem_u32(sA) + (w >> 3) * (MT_M * 128) + r * 128 + (((w & 7) ^ (r & 7)) << 4);
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(h[0]), "r"(h[1]), "r"(h[2]), "r"(h[3])
                     : "memory");
      }
    }
  }
}

// TMA warp: depth chunk c of the 96 text rows of pass `pass` into stage s, once the stage is free.  Advances (s, phase).
__device__ __forceinline__ void mt_text_stage(const CUtensorMap &tmT, uint8_t *sB, uint32_t b_full, uint32_t b_empty, int c,
                                              int pass, int &s, uint32_t &phase) {
  constexpr int B_BYTES = MT_NW * 128;
  mbar_wait(b_empty + 8 * s, phase ^ 1);
  if (elect_one()) {
    mbar_expect_tx(b_full + 8 * s, (uint32_t)B_BYTES);
    tma_load_2d(smem_u32(sB + s * B_BYTES), &tmT, b_full + 8 * s, c * 64, pass * MT_NW);
  }
  __syncwarp();
  if (++s == MT_BSTAGES) { s = 0; phase ^= 1; }
}

// wgmma warpgroup g: its 64 rows of sA times one 96-column text pass, chunk by chunk from the TMA stages, added to acc
// (zeroed by the caller; the fragment layout of tc_ptx.cuh).  Each stage is released to the TMA warp once read.  Advances (s, phase).
template <int NP>
__device__ __forceinline__ void mt_mma_pass(float (&acc)[MT_NW / 2], uint8_t *sA, uint8_t *sB, int g, int tid,
                                            uint32_t b_full, uint32_t b_empty, int &s, uint32_t &phase) {
  constexpr int B_BYTES = MT_NW * 128;
  for (int c = 0; c < NP; ++c) {
    mbar_wait(b_full + 8 * s, phase);
    const uint64_t da = gmma_desc(smem_u32(sA + c * (MT_M * 128) + g * 64 * 128)), db = gmma_desc(smem_u32(sB + s * B_BYTES));
    wgmma_fence();
#pragma unroll
    for (int h = 0; h < 4; ++h) {    // 64 fp16 per chunk = 4 K-steps of 16 (32 bytes each)
      wgmma_n64_f16<0, 0>(acc, da + 2 * h, db + 2 * h, 1u);
      wgmma_n32_f16<0, 0>(acc + 32, da + 2 * h, db + 2 * h + 512, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_hold(acc);
    if ((tid & 127) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(b_empty + 8 * s) : "memory");
    if (++s == MT_BSTAGES) { s = 0; phase ^= 1; }
  }
}

}  // namespace osb
