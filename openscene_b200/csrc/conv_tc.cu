// Sparse convolution on tensor cores: gathered rows -> shared memory -> wgmma -> register accumulators.
//
//   out[o,:] = epilogue( sum_k  in[nbr[k][o], :] @ W[k] )         (output-stationary, no atomics)
//
// Replaces MinkowskiConvolution / MinkowskiConvolutionTranspose forward (models/mink_unet.py:116-174)
// for channel counts that are multiples of 32, with BatchNorm(eval) / residual / ReLU / `ME.cat`
// folded in (mink_unet.py:50,114,147; BasicBlock).
//
// Numerics: fp32 operands are carried as split bf16 pairs (v = hi + lo) and every product is
// evaluated as hi*Whi + hi*Wlo + lo*Whi on bf16 wgmma with fp32 accumulation:
// ~2^-16 relative operand error, i.e. fp32-grade results at 1.5x the tensor time of one TF32 pass.
//
// One CTA = 128 output rows x NT output channels.  A pipeline stage holds one (offset k, 32-channel
// block) pair: A = 128 gathered rows x 128 B (128B swizzle; a missing neighbour is a zero-filled row),
// B = NT weight rows x 128 B (TMA tile load).
// Warpgroup 0 produces: warp w gathers rows [32w, 32w+32), warp 0 also loads the weight tiles.  Warpgroups
// 1 and 2 each multiply 64 rows of the tile (M64 x NT x K16 wgmma, accumulators in registers), then run the
// epilogue on them (affine/residual/ReLU -> split-bf16 or fp32 rows, through a swizzled staging tile).
// Two A paths are kept selectable (osb_tuning_set "tc_a_path"):
//   2 (default) cp.async.cg 16 B x 8 lanes per row, swizzled by hand, completion through
//               cp.async.mbarrier.arrive.noinc on the stage's full barrier;
//   0           one TMA row load per row (cross-check path; a missing row is an out-of-bounds row: zero fill).
#include "tc_ptx.cuh"
#include <algorithm>
#include <string>

namespace osb {

constexpr int TC_M = 128;          // rows per CTA
constexpr int TC_MAXK = 32;        // kernel offsets handled by this kernel (27, 8, 1)
constexpr int TC_THREADS = 384;    // producer warpgroup + two consumer warpgroups
constexpr int TC_A_BYTES = TC_M * 128;
constexpr int TC_STG_BYTES = 8 * 2048;   // epilogue staging: 8 consumer warps x (16 rows x 128 B)

struct ConvTcParams {
  const int32_t *nbr;
  int64_t n_out;
  int K, nb0, nb1;
  int n_src0, n_src1;
  int cout, cout_pad, nt, stages;
  const float *scale, *shift;
  const uint8_t *res;
  int relu;
  uint8_t *out_split;
  float *out_f32;
  const int32_t *out_row_map;
  int use_cpasync;       // A path: 1 = cp.async gathers, 0 = TMA row loads
  int nsplit;            // > 1: blockIdx.z handles a contiguous chunk of the (offset, channel-block) stage sequence
  float *partial;        // [nsplit][n_out][cout_pad] raw accumulators (nsplit > 1)
  const uint8_t *src0_ptr, *src1_ptr;   // raw bases (L2 prefetch of a later tile's own rows)
  int pf_dist;           // tiles ahead to prefetch into L2 (0 = off; only when input rows == output rows)
  const int32_t *cmap;   // dense transposed conv: per column block k = col / cmap_cout, tile row o goes to row cmap[k*n_out + o] (-1: drop)
  int cmap_cout;         //   ... and to column col % cmap_cout; outputs then have cmap_cout channels per row
  int lazy_idx;          // A producers read the kernel map per offset from global memory; no index prologue, all K offsets run
  int pdl;               // launched with programmatic stream serialization (see osb_conv_fwd_tc flags)
  int dbg_skip;          // tuning only: bit0 = no A gathers, bit1 = no B loads, bit2 = no main loop, bit3 = no stores
  long long *dbg_clock;  // tuning only: per-CTA timestamps [gridDim.x][8] (may be NULL)
};

// ------------------------------------------------------------------------------------ the kernel
template <int NCH>   // NT = 32 * NCH output channels per CTA
__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv_tc(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
          const __grid_constant__ CUtensorMap tmB, const ConvTcParams p) {
  constexpr int NT = 32 * NCH;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stage_bytes = TC_A_BYTES + NT * 128;
  const uint32_t stg_base = smem_u32(smem + p.stages * stage_bytes);
  uint8_t *aux = smem + p.stages * stage_bytes + TC_STG_BYTES;
  int32_t *s_nbr = reinterpret_cast<int32_t *>(aux);                        // [K][128]
  float *s_scale = reinterpret_cast<float *>(aux + (p.lazy_idx ? 0 : p.K * TC_M * 4));   // [nt]
  float *s_shift = s_scale + 256;                                           // [nt]
  uint64_t *bars = reinterpret_cast<uint64_t *>(s_shift + 256);             // full[8], empty[8]
  uint32_t *s_misc = reinterpret_cast<uint32_t *>(bars + 16);               // [0] kmask

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (p.pdl) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // the next kernel may start its prologue
  if (p.dbg_clock && tid == 0) { p.dbg_clock[blockIdx.x * 8 + 0] = clock64(); unsigned sm; asm("mov.u32 %0, %%smid;" : "=r"(sm)); p.dbg_clock[blockIdx.x * 8 + 7] = sm; }
  const int64_t row0 = (int64_t)blockIdx.x * TC_M;
  const int n0 = blockIdx.y * NT;
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + 8);

  if (tid == 32) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA0) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA1) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
  }
  if (tid == 0) {
    const uint32_t full_count = p.use_cpasync ? 1 + 128 : 1;     // B producer (+ 128 cp.async A producers)
    // empty: one arrival per consumer warpgroup
    for (int s = 0; s < p.stages; ++s) { mbar_init(full0 + 8 * s, full_count); mbar_init(empty0 + 8 * s, 2); }
    s_misc[0] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();   // s_misc[0] = 0 visible before the atomics below

  // ---- prologue: neighbour rows of this tile -> smem, bit mask of offsets that touch the tile.
  // All loads of a thread are issued before any is consumed (11 = ceil(32*128/384) independent loads).
  if (!p.lazy_idx) {
    constexpr int PRO = (TC_MAXK * TC_M + TC_THREADS - 1) / TC_THREADS;
    int32_t idx[PRO];
    const int total = p.K * TC_M;
#pragma unroll
    for (int j = 0; j < PRO; ++j) {
      const int e = tid + j * TC_THREADS;
      idx[j] = -1;
      if (e < total) {
        const int64_t o = row0 + (e & 127);
        if (o < p.n_out) idx[j] = p.nbr ? __ldg(p.nbr + (int64_t)(e >> 7) * p.n_out + o) : (int32_t)o;
      }
    }
    uint32_t mymask = 0;
#pragma unroll
    for (int j = 0; j < PRO; ++j) {
      const int e = tid + j * TC_THREADS;
      if (e < total) {
        s_nbr[e] = idx[j];
        if (idx[j] >= 0) mymask |= 1u << (e >> 7);
      }
    }
    mymask = __reduce_or_sync(0xffffffffu, mymask);
    if (lane == 0 && mymask) atomicOr(&s_misc[0], mymask);
  }
  for (int n = tid; n < NT; n += TC_THREADS) {
    const int c = n0 + n;
    const int cc = p.cmap ? c % p.cmap_cout : c;
    s_scale[n] = (p.scale && c < p.cout) ? __ldg(p.scale + cc) : 1.f;
    s_shift[n] = (p.shift && c < p.cout) ? __ldg(p.shift + cc) : 0.f;
  }
  __syncthreads();
  // Everything above touched only launch-invariant data (kernel map, BN constants).  The activations, the residual
  // and the shared split workspace belong to the previous kernel in the stream: wait for it to finish and flush.
  // PDL pre-wait reads: nbr[K][n_out], scale[cout], shift[cout]
  if (p.pdl) asm volatile("griddepcontrol.wait;" ::: "memory");
  const uint32_t kmask = (p.dbg_skip & 4) ? 0u : (p.lazy_idx ? (p.K >= 32 ? 0xffffffffu : ((1u << p.K) - 1u)) : s_misc[0]);
  if (p.dbg_clock && tid == 0) p.dbg_clock[blockIdx.x * 8 + 1] = clock64();
  const int nb = p.nb0 + p.nb1;
  // stage sequence of this tile = (valid offsets in ascending k) x (channel blocks); split mode takes a chunk
  const int n_stage_all = __popc(kmask) * nb;
  int t_begin = 0, t_end = n_stage_all;
  if (p.nsplit > 1) {
    const int per = (n_stage_all + p.nsplit - 1) / p.nsplit;
    t_begin = min((int)blockIdx.z * per, n_stage_all);
    t_end = min(t_begin + per, n_stage_all);
  }

  if (warp < 4) {
    // ============ producers: warp w gathers rows [32w, 32w+32) of every stage; warp 0 also loads the weight tiles ============
    const int w = warp;
    if (warp == 0 && p.pf_dist > 0 && blockIdx.y == 0 && blockIdx.z == 0 && elect_one()) {
      // Stride-1 convolutions read mostly the rows around their own tile (Morton order): pull the rows of the
      // tile that will run ~one wave later into L2 now, so its gathers do not wait on compulsory DRAM misses.
      const int64_t r0 = ((int64_t)blockIdx.x + p.pf_dist) * TC_M;
      if (r0 < p.n_out) {
        const int64_t nrows = min((int64_t)TC_M, p.n_out - r0);
        const uint32_t b0 = (uint32_t)(nrows * p.nb0 * 128);
        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.src0_ptr + r0 * p.nb0 * 128), "r"(b0) : "memory");
        if (p.nb1) {
          const uint32_t b1 = (uint32_t)(nrows * p.nb1 * 128);
          asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.src1_ptr + r0 * p.nb1 * 128), "r"(b1) : "memory");
        }
      }
    }
    __syncwarp();
    const int j = lane & 7, q = lane >> 3;
    int s = 0;
    uint32_t phase = 0;
    int t = 0;
    // lazy mode: this thread's 8 row indices of offset k come straight from the kernel map (L2), prefetched one
    // offset ahead so that the load latency hides behind the copies of the current offset
    auto fetch = [&](int k, int32_t (&r)[8]) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int64_t o = row0 + w * 32 + 4 * i + q;
        r[i] = (o < p.n_out) ? (p.nbr ? __ldg(p.nbr + (int64_t)k * p.n_out + o) : (int32_t)o) : -1;
      }
    };
    int32_t rnext[8];
    if (p.lazy_idx && kmask) fetch(__ffs(kmask) - 1, rnext);
    for (uint32_t km = kmask; km; km &= km - 1) {
      const int k = __ffs(km) - 1;
      int32_t ridx[8];
      if (p.lazy_idx) {
#pragma unroll
        for (int i = 0; i < 8; ++i) ridx[i] = rnext[i];
        const uint32_t rest = km & (km - 1);
        if (rest) fetch(__ffs(rest) - 1, rnext);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) ridx[i] = s_nbr[k * TC_M + w * 32 + 4 * i + q];
      }
      for (int cb = 0; cb < nb; ++cb, ++t) {
        if (t < t_begin || t >= t_end) continue;
        mbar_wait(empty0 + 8 * s, phase ^ 1);
        const uint32_t fb = full0 + 8 * s;
        const uint32_t a_base = smem_u32(smem + s * stage_bytes);
        if (warp == 0 && elect_one()) {
          uint32_t bytes = (uint32_t)stage_bytes;        // A (TMA row path) + B bytes of this stage
          if ((p.dbg_skip & 1) || p.use_cpasync) bytes -= TC_A_BYTES;
          if (p.dbg_skip & 2) bytes -= NT * 128;
          mbar_expect_tx(fb, bytes);
          if (!(p.dbg_skip & 2)) tma_load_2d(a_base + TC_A_BYTES, &tmB, fb, cb * 64, k * p.cout_pad + n0);
        }
        __syncwarp();
        const bool first = cb < p.nb0;
        if (p.use_cpasync) {
          // 8 lanes cover one 128-byte row line (one L2 line per 8 lanes), 4 rows per warp instruction, 8 instructions
          // per stage; the destination carries the 128B swizzle (chunk ^ (row & 7)).
          const uint8_t *src = first ? p.src0_ptr : p.src1_ptr;
          const int64_t row_bytes = (int64_t)(first ? p.nb0 : p.nb1) * 128;
          const int col_byte = (first ? cb : cb - p.nb0) * 128 + j * 16;
          const uint32_t a_dst = a_base + (w * 32 + q) * 128;
          if (!(p.dbg_skip & 1)) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int m7 = (4 * i + q) & 7;
              const bool valid = ridx[i] >= 0;
              const uint8_t *sp = valid ? src + (int64_t)ridx[i] * row_bytes + col_byte : src;
              cp_async16(a_dst + i * 512 + ((j ^ m7) << 4), sp, valid ? 16u : 0u);      // size 0 -> zero fill
            }
          }
          cp_async_arrive_noinc(fb);
        } else if (!(p.dbg_skip & 1)) {
          // one TMA row load per row; a missing row reads one past the last row: hardware zero fill
          const CUtensorMap *tm = first ? &tmA0 : &tmA1;
          const int col = (first ? cb : cb - p.nb0) * 64;
          const int oob = first ? p.n_src0 : p.n_src1;
#pragma unroll
          for (int rr = 0; rr < 32; ++rr) {
            const int r = __shfl_sync(0xffffffffu, ridx[rr >> 2], 8 * (rr & 3));   // row rr = 4i + q is held by lanes 8q..8q+7
            if (lane == 0) tma_load_2d(a_base + (w * 32 + rr) * 128, tm, fb, col, r >= 0 ? r : oob);
          }
        }
        if (++s == p.stages) { s = 0; phase ^= 1; }
      }
    }
    if (p.dbg_clock && tid == 0) p.dbg_clock[blockIdx.x * 8 + 2] = clock64();     // producers done issuing
  } else {
    // ============ consumers: warpgroup g multiplies tile rows [64g, 64g+64), then runs their epilogue ============
    const int g = (warp >> 2) - 1;
    float acc[16 * NCH];
#pragma unroll
    for (int i = 0; i < 16 * NCH; ++i) acc[i] = 0.f;
    int s = 0, s_prev = -1;
    uint32_t phase = 0;
    for (int t = t_begin; t < t_end; ++t) {
      mbar_wait(full0 + 8 * s, phase);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // cp.async (generic proxy) writes -> wgmma reads
      const uint32_t a_addr = smem_u32(smem + s * stage_bytes);
      wgmma_fence();
      wg_split_mma<NCH>(acc, gmma_desc(a_addr + g * 64 * 128), gmma_desc(a_addr + TC_A_BYTES));
      wgmma_commit();
      wgmma_wait<1>();                                               // the previous stage's wgmmas have retired: free it
      if (s_prev >= 0 && (tid & 127) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(empty0 + 8 * s_prev) : "memory");
      s_prev = s;
      if (++s == p.stages) { s = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_hold(acc);
    if (p.dbg_clock && tid == 128) p.dbg_clock[blockIdx.x * 8 + 3] = clock64();     // accumulator ready
    // Rows of this warp: tile rows [64g + 16(warp%4), +16).  Global traffic goes through a 2 KB staging tile per warp in
    // the 128B-swizzled layout, so that every global load / store instruction moves 4 full 128-byte lines.
    const bool no_store = (p.dbg_skip & 8) != 0;
    const uint32_t stg = stg_base + (uint32_t)(warp - 4) * 2048u;
    const int64_t wrow0 = row0 + 64 * g + 16 * (warp & 3);         // first global row of this warp
    const int cq = 2 * (lane & 3);
    auto plain_row = [&](int r) -> int64_t { return (!no_store && wrow0 + r < p.n_out) ? wrow0 + r : -1; };
#pragma unroll
    for (int cbo = 0; cbo < NCH; ++cbo) {
      float *y = acc + 16 * cbo;
      const int c0 = n0 + cbo * 32;              // first output channel of this 32-block
      if (p.nsplit > 1) {                        // raw partial sums; k_conv_finish reduces + applies the epilogue
        frag_stage_f32(stg, y, lane);
        __syncwarp();
        stage_flush(stg, reinterpret_cast<uint8_t *>(p.partial + (int64_t)blockIdx.z * p.n_out * p.cout_pad), (int64_t)p.cout_pad * 4,
                    (int64_t)c0 * 4, lane, plain_row);
        __syncwarp();
        continue;
      }
      if (c0 >= p.cout) continue;               // warp-uniform
      if (p.scale != nullptr) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int col = cbo * 32 + 8 * i + cq + (e & 1);
            y[4 * i + e] = fmaf(y[4 * i + e], s_scale[col], s_shift[col]);
          }
      }
      if (p.res) {                               // residual tile: coalesced load -> staging -> own fragment
        stage_load(stg, p.res, wrow0, p.n_out, (int64_t)p.cout * 4, (int64_t)(c0 >> 5) * 128, lane);
        __syncwarp();
        frag_add_split(stg, y, lane);
        __syncwarp();
      }
      if (p.relu) {
#pragma unroll
        for (int e = 0; e < 16; ++e) y[e] = fmaxf(y[e], 0.f);
      }
      int oc0 = c0;                                  // first output channel of this block in the destination row
      int out_c = p.cout;                            // channels per destination row
      int kch = 0;
      if (p.cmap) {                                  // dense transposed conv: this column block belongs to child kch
        kch = c0 / p.cmap_cout;
        oc0 = c0 - kch * p.cmap_cout;
        out_c = p.cmap_cout;
      }
      auto cmap_row = [&](int r) -> int64_t {
        return (!no_store && wrow0 + r < p.n_out) ? (int64_t)__ldg(p.cmap + (int64_t)kch * p.n_out + wrow0 + r) : -1;
      };
      if (p.out_split) {
        frag_stage_split(stg, y, lane);
        __syncwarp();
        if (p.cmap) stage_flush(stg, p.out_split, (int64_t)out_c * 4, (int64_t)(oc0 >> 5) * 128, lane, cmap_row);
        else stage_flush(stg, p.out_split, (int64_t)out_c * 4, (int64_t)(oc0 >> 5) * 128, lane, plain_row);
        __syncwarp();
      }
      if (p.out_f32) {
        frag_stage_f32(stg, y, lane);
        __syncwarp();
        uint8_t *base = reinterpret_cast<uint8_t *>(p.out_f32);
        if (p.cmap) stage_flush(stg, base, (int64_t)out_c * 4, (int64_t)oc0 * 4, lane, cmap_row);
        else if (p.out_row_map)
          stage_flush(stg, base, (int64_t)out_c * 4, (int64_t)oc0 * 4, lane, [&](int r) -> int64_t {
            return (!no_store && wrow0 + r < p.n_out) ? (int64_t)__ldg(p.out_row_map + wrow0 + r) : -1;
          });
        else stage_flush(stg, base, (int64_t)out_c * 4, (int64_t)oc0 * 4, lane, plain_row);
        __syncwarp();
      }
    }
  }
  if (p.dbg_clock && tid == 128) p.dbg_clock[blockIdx.x * 8 + 4] = clock64();     // epilogue stores issued
}

// ------------------------------------------------------------------ split-mode finish kernel
// out = epilogue( sum_z partial[z] ): one thread per (row, 8 channels)
__global__ void k_conv_finish(const float *__restrict__ partial, int nsplit, int64_t n_out, int cout, int cout_pad,
                              const float *__restrict__ scale, const float *__restrict__ shift,
                              const uint8_t *__restrict__ res, int relu, uint8_t *__restrict__ out_split,
                              float *__restrict__ out_f32, const int32_t *__restrict__ out_row_map, int pdl) {
  if (pdl) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    // PDL pre-wait reads: none
    asm volatile("griddepcontrol.wait;" ::: "memory");           // partials come from the k_conv_tc launch just before
  }
  const int groups = cout / 8;
  const int64_t total = n_out * groups;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = e / groups;
    const int c0 = (int)(e - o * groups) * 8;
    float y[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int z = 0; z < nsplit; ++z) {
      const float4 *pp = reinterpret_cast<const float4 *>(partial + ((int64_t)z * n_out + o) * cout_pad + c0);
      const float4 a = __ldg(pp), b = __ldg(pp + 1);
      y[0] += a.x; y[1] += a.y; y[2] += a.z; y[3] += a.w; y[4] += b.x; y[5] += b.y; y[6] += b.z; y[7] += b.w;
    }
    if (scale) {
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = fmaf(y[j], __ldg(scale + c0 + j), __ldg(shift + c0 + j));
    }
    const int64_t off = o * (int64_t)cout * 4 + split_off_hi(c0);
    if (res) {
      const uint4 hq = __ldg(reinterpret_cast<const uint4 *>(res + off)), lq = __ldg(reinterpret_cast<const uint4 *>(res + off + 64));
      const __nv_bfloat16 *hh = reinterpret_cast<const __nv_bfloat16 *>(&hq);
      const __nv_bfloat16 *ll = reinterpret_cast<const __nv_bfloat16 *>(&lq);
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] += join_bf16(hh[j], ll[j]);
    }
    if (relu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = fmaxf(y[j], 0.f);
    }
    if (out_split) {
      __align__(16) __nv_bfloat16 hh[8], ll[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) split_bf16(y[j], hh[j], ll[j]);
      *reinterpret_cast<uint4 *>(out_split + off) = *reinterpret_cast<const uint4 *>(hh);
      *reinterpret_cast<uint4 *>(out_split + off + 64) = *reinterpret_cast<const uint4 *>(ll);
    }
    if (out_f32) {
      const int64_t orow = out_row_map ? (int64_t)__ldg(out_row_map + o) : o;
      float4 *op = reinterpret_cast<float4 *>(out_f32 + orow * cout + c0);
      op[0] = make_float4(y[0], y[1], y[2], y[3]);
      op[1] = make_float4(y[4], y[5], y[6], y[7]);
    }
  }
}

// --------------------------------------------------------------------------- weight packing
__global__ void k_pack_weights(const float *__restrict__ w, int K, int cin, int cout, int cout_pad, int transpose_w,
                               uint8_t *__restrict__ wpack) {
  const int64_t total = (int64_t)K * cout_pad * cin;
  const int64_t sk = (int64_t)cin * cout, sn = transpose_w ? cin : 1, sc = transpose_w ? 1 : cout;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x)
    pack_weight_elem(w, sk, sn, sc, cin, cout, cout_pad, e, wpack);
}

// --------------------------------------------------------------------------- host side
static PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

// 2-D tensor [rows, cols_elems] of 2-byte elements with row pitch cols_elems*2 bytes; box {64 elems, box_rows}; 128B swizzle
int make_tmap_2b(CUtensorMap *tm, const void *base, uint64_t cols_elems, uint64_t rows, uint32_t box_rows, int is_f16) {
  auto enc = get_encode();
  OSB_CHECK(enc != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
  cuuint64_t gdim[2] = {cols_elems, rows};
  cuuint64_t gstride[1] = {cols_elems * 2};
  cuuint32_t box[2] = {64, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(tm, is_f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(base),
                   gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  OSB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d) base=%p cols=%llu rows=%llu box_rows=%u", (int)r, base,
            (unsigned long long)cols_elems, (unsigned long long)rows, box_rows);
  return 0;
}
static int make_tmap(CUtensorMap *tm, const void *base, uint64_t cols_elems, uint64_t rows, uint32_t box_rows) {
  return make_tmap_2b(tm, base, cols_elems, rows, box_rows, 0);
}

static int g_tc_a_path = 2;                 // A operand path: 2 = cp.async (default), 0 = TMA row loads
static int g_tc_smem_budget = 227 * 1024;   // per CTA: the register file holds one 384-thread CTA per SM
static int g_tc_dbg_skip = 0;
static int g_tc_force_split = 0;            // 0 = heuristic, >0 = forced nsplit (1 disables)
static int g_tc_target_ctas = 132;          // split small launches until ~one CTA per SM (H100 SXM: 132 SMs)
static int g_tc_pf_dist = 0;
static int g_tc_small_nt = 0;              // > 0: N tile used when the launch has few row tiles (tuning)
static int g_tc_small_rows = 5120;
static int g_tc_min_stages = 3;
static int g_tc_lazy = 1;                  // cp.async path: per-offset index fetch instead of the smem index prologue
static long long *g_tc_dbg_clock = nullptr;

// knobs of this kernel behind osb_tuning_set (conv_chain.cu); returns false for names it does not own
bool conv_tc_tuning(const char *name, int64_t v) {
  const std::string n(name);
  if (n == "tc_a_path") g_tc_a_path = (int)v;                 // 2 = cp.async (default), 0 = TMA row loads
  else if (n == "tc_smem_budget") g_tc_smem_budget = (int)v;  // per CTA
  else if (n == "tc_dbg_skip") g_tc_dbg_skip = (int)v;
  else if (n == "tc_force_split") g_tc_force_split = (int)v;
  else if (n == "tc_target_ctas") g_tc_target_ctas = (int)v;
  else if (n == "tc_pf_dist") g_tc_pf_dist = (int)v;
  else if (n == "tc_small_nt") g_tc_small_nt = (int)v;
  else if (n == "tc_min_stages") g_tc_min_stages = (int)v;
  else if (n == "tc_lazy") g_tc_lazy = (int)v;
  else if (n == "tc_dbg_clock") g_tc_dbg_clock = (long long *)(intptr_t)v;
  else return false;
  return true;
}

}  // namespace osb

using namespace osb;

static inline int choose_nt(int64_t n_out, int cp);
static inline int cout_pad_of(int cout) { return cout <= 256 ? (cout + 15) / 16 * 16 : (cout + 255) / 256 * 256; }

static inline int choose_nt(int64_t n_out, int cp) {
  int nt = cp <= 256 ? cp : 256;
  if (g_tc_small_nt > 0 && n_out <= g_tc_small_rows && nt > g_tc_small_nt && cp % g_tc_small_nt == 0) nt = g_tc_small_nt;
  return nt;
}

extern "C" {

// bytes of caller-provided scratch osb_conv_fwd_tc may need for this shape (0 = none)
size_t osb_conv_tc_workspace_bytes(int64_t n_out, int32_t K, int32_t cin, int32_t cout) {
  if (n_out <= 0 || K < 1 || cin < 32 || cout <= 0) return 0;     // shapes osb_conv_fwd_tc rejects: nothing to reserve
  const int cp = cout_pad_of(cout);
  const int nt = choose_nt(n_out, cp);
  const int64_t ctas = ceil_div(n_out, TC_M) * (cp / nt);
  int nsplit = g_tc_force_split > 0 ? g_tc_force_split : (int)(g_tc_target_ctas / ctas);
  nsplit = std::max(1, std::min(nsplit, std::min(32, K * (cin / 32))));
  return nsplit > 1 ? (size_t)nsplit * n_out * cp * sizeof(float) : 0;
}

size_t osb_conv_packed_weight_bytes(int32_t K, int32_t cin, int32_t cout) {
  return (size_t)K * cout_pad_of(cout) * cin * 4;
}

int osb_conv_pack_weights(const float *w, int32_t K, int32_t cin, int32_t cout, int32_t transpose_w, void *wpack,
                          void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(K >= 1 && cin % 32 == 0 && cin > 0 && cout > 0, "osb_conv_pack_weights: cin (%d) must be a multiple of 32", cin);
  const int cp = cout_pad_of(cout);
  const int64_t total = (int64_t)K * cp * cin;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(total, 256), 132 * 32);
  k_pack_weights<<<grid, 256, 0, stream>>>(w, K, cin, cout, cp, transpose_w, (uint8_t *)wpack);
  OSB_LAUNCH_CHECK();
  return 0;
}

static int conv_fwd_tc_impl(const void *src0, int32_t c0, int64_t n_src0, const void *src1, int32_t c1, int64_t n_src1,
                            const int32_t *nbr, int64_t n_out, int32_t K, const void *wpack, int32_t cout, const float *scale,
                            const float *shift, const void *res, int32_t relu, void *out_split, float *out_f32,
                            const int32_t *out_row_map, void *ws, size_t ws_bytes, int32_t flags, void *stream_,
                            const int32_t *cmap, int32_t cmap_cout);

int osb_conv_fwd_tc(const void *src0, int32_t c0, int64_t n_src0, const void *src1, int32_t c1, int64_t n_src1,
                    const int32_t *nbr, int64_t n_out, int32_t K, const void *wpack, int32_t cout, const float *scale,
                    const float *shift, const void *res, int32_t relu, void *out_split, float *out_f32,
                    const int32_t *out_row_map, void *ws, size_t ws_bytes, int32_t flags, void *stream_) {
  return conv_fwd_tc_impl(src0, c0, n_src0, src1, c1, n_src1, nbr, n_out, K, wpack, cout, scale, shift, res, relu, out_split,
                          out_f32, out_row_map, ws, ws_bytes, flags, stream_, nullptr, 0);
}

// Transposed stride-2 convolution as a dense GEMM over the COARSE rows: z[o, k*cout + c] = sum_ci x[o, ci] W[k][ci][c]
// (wpack = osb_conv_pack_weights of the [1, cin, kvol*cout] matrix), whose epilogue sends column block k of coarse row o
// to the fine row down_nbr[k*n_coarse + o] (the stride-2 kernel map of the matching strided conv; -1 = that child does
// not exist).  Every fine row has exactly one (parent, k), so each output row is written exactly once.
int osb_convtr_fwd_tc(const void *src, int32_t cin, int64_t n_coarse, const int32_t *down_nbr, int32_t kvol, const void *wpack,
                      int32_t cout, const float *scale, const float *shift, int32_t relu, void *out_split, float *out_f32,
                      int32_t flags, void *stream_) {
  OSB_CHECK(down_nbr != nullptr && kvol >= 1 && cout % 32 == 0, "osb_convtr_fwd_tc: bad arguments");
  return conv_fwd_tc_impl(src, cin, n_coarse, nullptr, 0, 0, nullptr, n_coarse, 1, wpack, kvol * cout, scale, shift, nullptr, relu,
                          out_split, out_f32, nullptr, nullptr, 0, flags, stream_, down_nbr, cout);
}

static int conv_fwd_tc_impl(const void *src0, int32_t c0, int64_t n_src0, const void *src1, int32_t c1, int64_t n_src1,
                            const int32_t *nbr, int64_t n_out, int32_t K, const void *wpack, int32_t cout, const float *scale,
                            const float *shift, const void *res, int32_t relu, void *out_split, float *out_f32,
                            const int32_t *out_row_map, void *ws, size_t ws_bytes, int32_t flags, void *stream_,
                            const int32_t *cmap, int32_t cmap_cout) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(src0 && c0 > 0 && c0 % 32 == 0 && c1 >= 0 && c1 % 32 == 0, "osb_conv_fwd_tc: channel counts must be multiples of 32 (c0=%d c1=%d)", c0, c1);
  OSB_CHECK((c1 == 0) == (src1 == nullptr), "osb_conv_fwd_tc: src1 / c1 mismatch");
  OSB_CHECK(K >= 1 && K <= TC_MAXK, "osb_conv_fwd_tc: K=%d not supported (<= %d)", K, TC_MAXK);
  OSB_CHECK(nbr != nullptr || K == 1, "osb_conv_fwd_tc: identity map needs K == 1");
  OSB_CHECK(n_out > 0 && n_src0 > 0 && n_src0 < (1ll << 31) && n_src1 < (1ll << 31), "osb_conv_fwd_tc: bad row counts");
  OSB_CHECK(cout % 32 == 0 && cout > 0, "osb_conv_fwd_tc: cout (%d) must be a multiple of 32", cout);
  OSB_CHECK(out_split || out_f32, "osb_conv_fwd_tc: no output given");
  OSB_CHECK((scale == nullptr) == (shift == nullptr), "osb_conv_fwd_tc: scale and shift go together");
  const int cin = c0 + c1;
  const int cp = cout_pad_of(cout);
  ConvTcParams p{};
  p.nt = choose_nt(n_out, cp);
  OSB_CHECK(g_tc_a_path == 2 || g_tc_a_path == 0, "osb_conv_fwd_tc: A path %d does not exist (2 = cp.async, 0 = TMA rows)", g_tc_a_path);
  const int stage_bytes = TC_A_BYTES + p.nt * 128;
  // lazy index fetch pays off on multi-wave launches (every tile touches all K offsets, the smem prologue is pure set-up
  // cost); on single-wave levels skipping empty (tile, offset) stages wins
  const int lazy = (g_tc_a_path == 2 && g_tc_lazy == 1 && ceil_div(n_out, TC_M) >= 4 * 132) || g_tc_lazy == 2 ? 1 : 0;
  const int aux_bytes = TC_STG_BYTES + (lazy ? 0 : K * TC_M * 4) + 2 * 256 * 4 + 16 * 8 + 64;
  const int seq = K * (cin / 32);                                         // stages one tile runs through (upper bound)
  int stages = (g_tc_smem_budget - 1024 - aux_bytes) / stage_bytes;      // what the budget holds (default: the whole SM) ...
  if (stages < g_tc_min_stages && !(stages == 2 && seq <= 4))            // ... unless that is too few for a longer sequence
    stages = (226 * 1024 - 1024 - aux_bytes) / stage_bytes;
  stages = std::max(2, std::min(8, std::min(stages, std::max(2, seq))));
  const size_t smem_bytes = (size_t)stages * stage_bytes + aux_bytes + 1024;
  OSB_CHECK(smem_bytes <= 227 * 1024, "osb_conv_fwd_tc: tile does not fit in shared memory");

  CUtensorMap tmA0, tmA1, tmB;
  if (make_tmap(&tmA0, src0, 2ull * c0, (uint64_t)n_src0, 1)) return 1;
  if (c1) { if (make_tmap(&tmA1, src1, 2ull * c1, (uint64_t)n_src1, 1)) return 1; }
  else tmA1 = tmA0;
  if (make_tmap(&tmB, wpack, 2ull * cin, (uint64_t)K * cp, (uint32_t)p.nt)) return 1;

  p.nbr = nbr; p.n_out = n_out; p.K = K; p.nb0 = c0 / 32; p.nb1 = c1 / 32;
  p.n_src0 = (int)n_src0; p.n_src1 = (int)n_src1;
  p.cout = cout; p.cout_pad = cp; p.stages = stages;
  p.scale = scale; p.shift = shift; p.res = (const uint8_t *)res; p.relu = relu;
  p.out_split = (uint8_t *)out_split; p.out_f32 = out_f32; p.out_row_map = out_row_map;
  p.use_cpasync = g_tc_a_path == 2 ? 1 : 0;
  p.dbg_skip = g_tc_dbg_skip;
  p.pdl = (flags & 1) ? 1 : 0;
  p.lazy_idx = lazy;
  p.cmap = cmap; p.cmap_cout = cmap_cout;
  p.dbg_clock = g_tc_dbg_clock;
  p.src0_ptr = (const uint8_t *)src0; p.src1_ptr = (const uint8_t *)src1;
  p.pf_dist = (n_src0 == n_out && (c1 == 0 || n_src1 == n_out) && (K & 1)) ? g_tc_pf_dist : 0;
  const size_t need = cmap ? 0 : osb_conv_tc_workspace_bytes(n_out, K, cin, cout);
  p.nsplit = 1;
  p.partial = nullptr;
  if (need > 0) {
    OSB_CHECK(ws != nullptr && ws_bytes >= need, "osb_conv_fwd_tc: workspace of %zu bytes required (got %zu)", need, ws_bytes);
    p.nsplit = (int)(need / ((size_t)n_out * cp * sizeof(float)));
    p.partial = (float *)ws;
  }

  dim3 grid((unsigned)ceil_div(n_out, TC_M), (unsigned)(cp / p.nt), (unsigned)p.nsplit);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
  cfg.attrs = attr; cfg.numAttrs = p.pdl ? 1 : 0;
  switch (p.nt / 32) {
#define OSB_TC_CASE(n)                                                 \
    case n:                                                            \
      OSB_SMEM_ATTR_ONCE(k_conv_tc<n>, 227 * 1024);                    \
      OSB_CUDA(cudaLaunchKernelEx(&cfg, k_conv_tc<n>, tmA0, tmA1, tmB, p)); \
      break;
    OSB_TC_CASE(1) OSB_TC_CASE(2) OSB_TC_CASE(3) OSB_TC_CASE(4) OSB_TC_CASE(5) OSB_TC_CASE(6) OSB_TC_CASE(7) OSB_TC_CASE(8)
#undef OSB_TC_CASE
    default: OSB_CHECK(false, "osb_conv_fwd_tc: N tile %d not supported", p.nt);
  }
  OSB_LAUNCH_CHECK();
  if (p.nsplit > 1) {
    const int64_t total = n_out * (cout / 8);
    const unsigned fgrid = (unsigned)std::min<int64_t>(ceil_div(total, 256), 132 * 8);
    cudaLaunchConfig_t fcfg{};
    fcfg.gridDim = dim3(fgrid); fcfg.blockDim = dim3(256); fcfg.dynamicSmemBytes = 0; fcfg.stream = stream;
    fcfg.attrs = attr; fcfg.numAttrs = p.pdl ? 1 : 0;
    OSB_CUDA(cudaLaunchKernelEx(&fcfg, k_conv_finish, (const float *)p.partial, p.nsplit, n_out, (int)cout, cp, scale, shift,
                                (const uint8_t *)res, (int)relu, (uint8_t *)out_split, out_f32, out_row_map, p.pdl));
    OSB_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
