// Persistent, plan-driven sparse convolution on tensor cores (wgmma; second generation of conv_tc.cu).
//
//   out[o,:] = epilogue( sum_k  in[nbr[k][o], :] @ W[k] )         (output-stationary, no atomics)
//
// One launch executes a LIST of convolution layers ("chain") described by ConvDesc records passed as kernel parameters.  The
// grid is one CTA per SM; every CTA owns a contiguous range of each layer's work units (unit = 128 output rows x one N tile x
// one split of the (offset, channel-block) stage sequence) and walks it with warp-specialised roles that never leave
// their loops between units:
//
//   warp 0       weight tiles: one cp.async.bulk per stage from the tile-major, pre-swizzled packing (no tensor map)
//   warps 1-3    gathered A rows: cp.async 16 B x 8 lanes per 128-byte row line, hand-applied 128B swizzle, the kernel
//                map read per offset straight from global memory, one slot of the warp ahead
//   warps 4-11   two consumer warpgroups: warpgroup g multiplies rows [64g, 64g+64) of every sub-tile of an item (wgmma,
//                accumulators in registers), then runs the epilogue on them: BN affine / residual / ReLU -> swizzled
//                staging tile -> full-line coalesced stores (split rows, fp32 rows, or raw split-K partials)
//
// Against conv_tc.cu:
//   * separate rings for gathered rows and weight tiles; the whole SM's shared memory belongs to one CTA;
//   * two 128-row sub-tiles share every weight tile (256 output rows per item) for N tiles of at most CH_MAX_PAIR_NT
//     columns: half the L2->SM weight stream;
//   * barrier set-up is paid once per CTA, not once per tile; work is split evenly over the SMs (no wave tail);
//   * split-K partials are reduced INSIDE the kernel after a grid barrier, and consecutive small layers (levels 2-4 of
//     the U-Net) run in one launch with grid barriers between dependent layers: no launch / finish-kernel boundaries.
//
// Numerics are those of conv_tc.cu: split-bf16 operands (v = hi + lo), hi*Whi + hi*Wlo + lo*Whi on bf16 wgmma,
// fp32 accumulation, deterministic (fixed-order) split-K reduction.
#include "tc_ptx.cuh"
#include <algorithm>
#include <cstring>
#include <string>

namespace osb {

constexpr int CH_THREADS = 384;                  // 12 warps (168 registers each): 1 weights, 3 gather, 2 consumer warpgroups
constexpr int CH_M = 128;                        // rows per sub-tile
constexpr int CH_A_BYTES = CH_M * 128;           // one row slot: 128 rows x one 32-channel block
constexpr int CH_STG_BYTES = 8 * 2048;           // epilogue staging: 8 consumer warps x (16 rows x 128 B)
constexpr int CH_SS_FLOATS = 768;                // folded BN constants kept in shared memory per layer (scale | shift)
constexpr int CH_MAX_SA = 12, CH_MAX_SB = 4;
// Warp roles.  Every producer role is ONE warp walking a dependent instruction chain, so its fixed cost per row slot
// (barrier wait, address set-up, arrival) is latency, not throughput.  Gather producers therefore own whole slots (ring slot
// s is always filled by warp s mod CH_A_WARPS, 32 copy instructions behind one wait / one arrival).
constexpr int CH_W_B = 0;                         // weight tiles
constexpr int CH_W_A = 1;                         // warps 1-3: gathered rows, one whole 128-row slot at a time each
constexpr int CH_A_WARPS = 3;
constexpr int CH_W_MMA = 4;                       // warps 4-11: two consumer warpgroups (wgmma + epilogue)
constexpr int CH_DESC_WORDS = 48;                // sizeof(ConvDesc) / 4
constexpr int CH_MAX_LAYERS = 16;                // layers per launch: the descriptors travel as kernel parameters (3 KB)

struct __align__(16) ConvDesc {
  const uint8_t *src0, *src1;      // split rows of the (up to) two sources ([src0 | src1] = ME.cat)
  const int32_t *nbr;              // [K][n_out] input row per (offset, output row), -1 = none; NULL = identity (K == 1)
  const uint8_t *wtiles;           // tile-major pre-swizzled weights (osb_conv_pack_weight_tiles)
  const float *scale, *shift;      // folded BatchNorm, or NULL
  const uint8_t *res;              // residual split rows [n_out, cout], or NULL
  uint8_t *out_split;              // split rows out, or NULL
  float *out_f32;                  // fp32 rows out, or NULL
  const int32_t *out_row_map;      // fp32 rows scattered: row o -> out_row_map[o]
  const int32_t *cmap;             // dense transposed conv: column block kch of row o -> fine row cmap[kch*n_out + o]
  float *partial;                  // [nsplit][n_out][cout_pad] raw accumulators (nsplit > 1)
  int64_t n_out;
  int K, nb0, nb1;
  int cout, cout_pad, nt, n_ntiles;
  int relu, cmap_cout, nsplit, m_tiles;
  int nsub_max;                    // sub-tiles per item that may share a weight tile: 2 when nt <= CH_MAX_PAIR_NT, else 1
  int barrier_before;              // grid barrier before this layer (it reads what an earlier layer of the launch wrote)
  int stages_per_split;            // ceil(K * (nb0 + nb1) / nsplit)
  int pad[8];
};
static_assert(sizeof(ConvDesc) == CH_DESC_WORDS * 4, "ConvDesc layout");
// The layer list lives in the kernel's parameter (constant) space: every field is a warp-uniform value to the compiler, so
// the roles keep their slot / descriptor arithmetic on the uniform datapath.
struct ChainArgs { ConvDesc d[CH_MAX_LAYERS]; };

__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// one non-blocking-ish probe of an mbarrier phase (true = complete).  Several probes issued back to back overlap their
// ~190-cycle round trips; a chain of mbar_wait calls pays them one after the other.
__device__ __forceinline__ uint32_t mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done;
}

// A wait that never completes must not hang the GPU: after ~2^24 probes the thread reports where it is stuck into the
// tuning buffer (if one is set; use pinned host memory so that the report survives the trap) and traps.
__device__ long long *g_chain_report = nullptr;
__device__ __noinline__ void chain_stuck(uint32_t bar, uint32_t parity, int tag, uint32_t it) {
  long long *r = g_chain_report;
  if (r && it == (1u << 20) + 1) {               // report once, keep waiting so that the other stuck roles can report too
    long long *o = r + 1 + 4 * ((blockIdx.x * 16 + (threadIdx.x >> 5)) % 1024);
    o[0] = ((long long)blockIdx.x << 32) | (threadIdx.x >> 5); o[1] = bar; o[2] = parity; o[3] = tag;
    r[0] = 1;
    __threadfence_system();
  }
  if (it > (1u << 23) || !r) __trap();
}
__device__ __forceinline__ void chain_wait(uint32_t bar, uint32_t parity, int tag) {
  for (uint32_t it = 0;; ++it) {
    if (mbar_try(bar, parity)) return;
    if (it > (1u << 20)) chain_stuck(bar, parity, tag, it);
  }
}

// wait of a role with slack (epilogue, weight producer): back off between polls so that the polling does not take issue slots
// from the roles on the critical path
__device__ __forceinline__ void mbar_wait_relaxed(uint32_t bar, uint32_t parity, unsigned sleep_ns) {
  uint32_t done = 0;
  for (uint32_t it = 0; !done; ++it) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (!done) {
      __nanosleep(sleep_ns);
      if (it > (1u << 24)) __trap();
    }
  }
}
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned *p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// no ordering of later accesses behind it: the thread stalls only where the value is used
__device__ __forceinline__ unsigned ld_relaxed_u32(const unsigned *p) {
  unsigned v;
  asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

// Sense-reversing grid barrier over {count, generation} in global memory (both zero before the first use ever; the
// barrier leaves count == 0 behind, so no host-side reset between launches).  Every CTA of the grid must be resident:
// the launch uses at most one CTA per SM.
__device__ __forceinline__ void grid_barrier(unsigned *gbar, unsigned &gen) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned old = atomicAdd(gbar, 1u);
    if (old == gridDim.x - 1) {
      gbar[0] = 0;
      __threadfence();
      atomicAdd(gbar + 1, 1u);
    } else {
      unsigned it = 0;
      while (ld_acquire_u32(gbar + 1) == gen) {
        if (++it > (1u << 24)) __trap();          // a CTA that never arrives must not hang the GPU
      }
    }
    __threadfence();
  }
  gen += 1;
  __syncthreads();
}

// keep a value in its register: stops the compiler from re-deriving shared-window addresses (S2R + shifts) in hot loops
#define CH_KEEP(x) asm volatile("" : "+r"(x))

// 16-byte global -> shared copy; `ignore` != 0 writes zeros instead (a missing neighbour row)
__device__ __forceinline__ void cp_async16_zfill(uint32_t dst, const void *src, uint32_t ignore) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %2, 0;\n\t"
      "cp.async.cg.shared.global [%0], [%1], 16, p;\n\t}"
      ::"r"(dst), "l"(src), "r"(ignore)
      : "memory");
}

// ------------------------------------------------------------------------------------ consumer: one item
// Rings and barriers of the CTA, as a consumer warpgroup sees them.
struct ChainRings {
  uint32_t a_ring, b_ring, bslot, sa, sb;
  uint32_t fullA, emptyA, fullB, emptyB;
};

// One item of consumer warpgroup g: rows [64g, 64g+64) of NSUB 128-row sub-tiles sharing each weight tile, N = 32 NCH
// columns, stages [t_begin, t_end).  Compile-time shapes keep the accumulators a fixed register set and every wgmma of a
// stage branch-free, so a stage's wgmmas stay in flight while the next stage's barriers are awaited; its slots are released
// one stage later (after wgmma_wait<1>).  Sub-tile s, 32-column block c accumulates in acc[16 (NCH s + c) ..].
template <int NCH, int NSUB>
__device__ __forceinline__ void chain_item(const ChainRings &R, const ConvDesc &E, const float *s_ss, uint32_t stgw, bool no_store,
                                           uint32_t &a_slot_io, uint32_t &a_phase_io,
                                        uint32_t &b_slot_io, uint32_t &b_phase_io, int t_begin, int t_end, int z, int nti, int m,
                                        int g, int warp, int lane) {
  float acc[NSUB * NCH * 16];
#pragma unroll
  for (int i = 0; i < NSUB * NCH * 16; ++i) acc[i] = 0.f;
  const bool leader = (threadIdx.x & 127) == 0;
  uint32_t a_slot = a_slot_io, a_phase = a_phase_io, b_slot = b_slot_io, b_phase = b_phase_io;   // ring positions, in registers
  uint32_t pa0 = 0, pa1 = 0, pb = 0;                 // slots of the previous stage, to release
  for (int t = t_begin; t < t_end; ++t) {
    uint32_t a1 = a_slot + 1u, ap1 = a_phase;
    if (a1 >= R.sa) { a1 -= R.sa; ap1 ^= 1u; }
    for (uint32_t it = 0;; ++it) {                   // all barriers of the stage probed together (overlapping round trips)
      uint32_t ok = mbar_try(R.fullB + 8 * b_slot, b_phase) & mbar_try(R.fullA + 8 * a_slot, a_phase);
      if (NSUB == 2) ok &= mbar_try(R.fullA + 8 * a1, ap1);
      if (ok) break;
      if (it > (1u << 26)) __trap();
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // cp.async (generic proxy) writes -> wgmma reads
    const uint64_t db = gmma_desc(R.b_ring + b_slot * R.bslot);
    wgmma_fence();
    wg_split_mma<NCH>(acc, gmma_desc(R.a_ring + a_slot * (uint32_t)CH_A_BYTES + (uint32_t)g * 64u * 128u), db);
    if (NSUB == 2) wg_split_mma<NCH>(acc + NCH * 16, gmma_desc(R.a_ring + a1 * (uint32_t)CH_A_BYTES + (uint32_t)g * 64u * 128u), db);
    wgmma_commit();
    wgmma_wait<1>();                                  // the previous stage's wgmmas have retired: release its slots
    if (leader && t > t_begin) {
      mbar_arrive(R.emptyA + 8 * pa0);
      if (NSUB == 2) mbar_arrive(R.emptyA + 8 * pa1);
      mbar_arrive(R.emptyB + 8 * pb);
    }
    pa0 = a_slot; pa1 = a1; pb = b_slot;
    a_slot += (uint32_t)NSUB;
    if (a_slot >= R.sa) { a_slot -= R.sa; a_phase ^= 1u; }
    if (++b_slot == R.sb) { b_slot = 0; b_phase ^= 1; }
  }
  wgmma_wait<0>();
  wgmma_hold(acc);
  a_slot_io = a_slot; a_phase_io = a_phase; b_slot_io = b_slot; b_phase_io = b_phase;
  if (leader && t_end > t_begin) {
    mbar_arrive(R.emptyA + 8 * pa0);
    if (NSUB == 2) mbar_arrive(R.emptyA + 8 * pa1);
    mbar_arrive(R.emptyB + 8 * pb);
  }
  // ---- epilogue of this warp's 16 rows of every sub-tile, one 32-column block at a time
  const int cq = 2 * (lane & 3);
#pragma unroll
  for (int s = 0; s < NSUB; ++s) {
    const int64_t wrow0 = (int64_t)(m + s) * CH_M + 64 * g + 16 * (warp & 3);   // first global row of this warp
    auto plain_row = [&](int r) -> int64_t { return (!no_store && wrow0 + r < E.n_out) ? wrow0 + r : -1; };
#pragma unroll
    for (int cbo = 0; cbo < NCH; ++cbo) {
      float *y = acc + 16 * (NCH * s + cbo);
      const int c0 = nti * E.nt + cbo * 32;           // first output channel of this 32-block
      if (E.nsplit > 1) {                             // raw partial sums; the reduce phase applies the epilogue
        frag_stage_f32(stgw, y, lane);
        __syncwarp();
        stage_flush(stgw, reinterpret_cast<uint8_t *>(E.partial + (int64_t)z * E.n_out * E.cout_pad), (int64_t)E.cout_pad * 4,
                    (int64_t)c0 * 4, lane, plain_row);
        __syncwarp();
        continue;
      }
      if (c0 >= E.cout) continue;                     // warp-uniform (padding columns)
      int oc0 = c0, out_c = E.cout, kch = 0;
      if (E.cmap) {                                   // dense transposed conv: this column block belongs to child kch
        kch = c0 / E.cmap_cout;
        oc0 = c0 - kch * E.cmap_cout;
        out_c = E.cmap_cout;
      }
      if (E.scale) {
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int col = oc0 + 8 * i + cq + (e & 1);
            y[4 * i + e] = fmaf(y[4 * i + e], s_ss[col], s_ss[CH_SS_FLOATS + col]);
          }
      }
      if (E.res) {                                    // residual tile: coalesced load -> staging -> own fragment
        stage_load(stgw, E.res, wrow0, E.n_out, (int64_t)E.cout * 4, (int64_t)(c0 >> 5) * 128, lane);
        __syncwarp();
        frag_add_split(stgw, y, lane);
        __syncwarp();
      }
      if (E.relu) {
#pragma unroll
        for (int e = 0; e < 16; ++e) y[e] = fmaxf(y[e], 0.f);
      }
      auto cmap_row = [&](int r) -> int64_t {
        return (!no_store && wrow0 + r < E.n_out) ? (int64_t)__ldg(E.cmap + (int64_t)kch * E.n_out + wrow0 + r) : -1;
      };
      if (E.out_split) {
        frag_stage_split(stgw, y, lane);
        __syncwarp();
        if (E.cmap) stage_flush(stgw, E.out_split, (int64_t)out_c * 4, (int64_t)(oc0 >> 5) * 128, lane, cmap_row);
        else stage_flush(stgw, E.out_split, (int64_t)out_c * 4, (int64_t)(oc0 >> 5) * 128, lane, plain_row);
        __syncwarp();
      }
      if (E.out_f32) {
        frag_stage_f32(stgw, y, lane);
        __syncwarp();
        uint8_t *base = reinterpret_cast<uint8_t *>(E.out_f32);
        if (E.cmap) stage_flush(stgw, base, (int64_t)out_c * 4, (int64_t)oc0 * 4, lane, cmap_row);
        else if (E.out_row_map)
          stage_flush(stgw, base, (int64_t)out_c * 4, (int64_t)oc0 * 4, lane, [&](int r) -> int64_t {
            return (!no_store && wrow0 + r < E.n_out) ? (int64_t)__ldg(E.out_row_map + wrow0 + r) : -1;
          });
        else stage_flush(stgw, base, (int64_t)out_c * 4, (int64_t)oc0 * 4, lane, plain_row);
        __syncwarp();
      }
    }
  }
}

// ------------------------------------------------------------------------------------ the kernel
__global__ void __launch_bounds__(CH_THREADS, 1)
k_conv_chain(const __grid_constant__ ChainArgs args, int n_layers, unsigned *gbar, int sa, int sb, int bslot, int flags,
             long long *dbg_clock) {
  extern __shared__ uint8_t smem_raw[];
  // All hot-loop addressing is done on 32-bit shared-window addresses computed once; the few generic accesses (descriptor,
  // BN constants) use pointers derived from smem_raw by an offset, so that the compiler keeps them in the shared space.
  const uint32_t raw_u32 = smem_u32(smem_raw);
  const uint32_t base_u32 = (raw_u32 + 1023u) & ~1023u;                      // 1024-byte aligned: 128B-swizzle atoms
  uint8_t *smem = smem_raw + (base_u32 - raw_u32);
  const uint32_t a_ring = base_u32;                                          // row slots
  const uint32_t b_ring = a_ring + (uint32_t)sa * CH_A_BYTES;                // weight slots (bslot is a multiple of 1024)
  const uint32_t stg_u32 = b_ring + (uint32_t)sb * (uint32_t)bslot;          // epilogue staging: 8 warps x 2 KB
  uint32_t a_ring_k = a_ring, b_ring_k = b_ring;
  CH_KEEP(a_ring_k); CH_KEEP(b_ring_k);
  uint8_t *aux = smem + (stg_u32 - base_u32) + CH_STG_BYTES;
  float *s_ss = reinterpret_cast<float *>(aux);                              // [scale x CH_SS_FLOATS | shift x CH_SS_FLOATS]
  uint64_t *bars = reinterpret_cast<uint64_t *>(s_ss + 2 * CH_SS_FLOATS);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (flags & 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (dbg_clock && tid == 0) dbg_clock[blockIdx.x * 32 + 0] = clock64();
  uint32_t fullA = smem_u32(bars), emptyA = fullA + 12 * 8, fullB = fullA + 24 * 8, emptyB = fullA + 28 * 8;
  CH_KEEP(fullA); CH_KEEP(emptyA); CH_KEEP(fullB); CH_KEEP(emptyB);

  if (tid == 0) {
    // fullA: the 32 lanes of the slot's warp; emptyA / emptyB: one arrival per consumer warpgroup
    for (int s = 0; s < sa; ++s) { mbar_init(fullA + 8 * s, 32); mbar_init(emptyA + 8 * s, 2); }
    for (int s = 0; s < sb; ++s) { mbar_init(fullB + 8 * s, 1); mbar_init(emptyB + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Everything above touched no data of an earlier kernel in the stream; from here on we read activations.
  // PDL pre-wait reads: none (the layer descriptors are launch parameters)
  if (flags & 1) asm volatile("griddepcontrol.wait;" ::: "memory");
  // The barrier generation is read behind the wait: the previous chain launch in the stream may still be running its own
  // barriers until then (a grid smaller than the SM count lets this launch's CTAs start beside it), and a generation read
  // too early lets this launch's barriers pass without waiting.  It is read before this launch's first barrier can complete;
  // the wait has made the previous launches' last value visible, so a relaxed load suffices and costs no stall before use.
  unsigned bar_gen = 0;
  if (tid == 0 && gbar) bar_gen = ld_relaxed_u32(gbar + 1);
  if (dbg_clock && tid == 0) dbg_clock[blockIdx.x * 32 + 1] = clock64();

  // pipeline state of this thread's role; persists over items and layers
  uint32_t a_slot = 0, a_phase = 0, b_slot = 0, b_phase = 0;
  uint32_t g_slot = 0;                             // gather producers: row slots the CTA has gone through before the current item
  uint32_t p_sl = (warp >= CH_W_A && warp < CH_W_A + CH_A_WARPS) ? (uint32_t)(warp - CH_W_A) : 0u, p_lapb = 0, p_par = 0;   // gather producers: my next ring slot, global index of slot 0 of its lap, lap parity

  for (int L = 0; L < n_layers; ++L) {
    __syncthreads();                                   // every role is done with the previous layer (and with s_ss)
    const ConvDesc *s_desc = &args.d[L];               // parameter space: uniform loads
    const int d_K = s_desc->K, d_nb0 = s_desc->nb0, d_nb1 = s_desc->nb1, d_nt = s_desc->nt, d_n_ntiles = s_desc->n_ntiles;
    const int d_m_tiles = s_desc->m_tiles, d_nsplit = s_desc->nsplit, d_nsub_max = s_desc->nsub_max, d_sps = s_desc->stages_per_split;
    const int64_t d_n_out = s_desc->n_out;
    {                                                  // folded BN constants of the layer -> shared memory
      const int nss = s_desc->cmap ? s_desc->cmap_cout : s_desc->cout;
      const float *sc = s_desc->scale, *sh = s_desc->shift;
      for (int c = tid; c < nss && c < CH_SS_FLOATS; c += CH_THREADS) {
        s_ss[c] = sc ? __ldg(sc + c) : 1.f;
        s_ss[CH_SS_FLOATS + c] = sh ? __ldg(sh + c) : 0.f;
      }
    }
    if (s_desc->barrier_before) {
      grid_barrier(gbar, bar_gen);                     // (only thread 0's copy of bar_gen is meaningful)
    } else {
      __syncthreads();
    }

    const int nb = d_nb0 + d_nb1;
    const int T = d_K * nb;                                            // stages of one full (offset, channel block) sweep
    const int64_t U = (int64_t)d_m_tiles * d_n_ntiles * d_nsplit;      // work units of the layer
    const int64_t u_begin = U * blockIdx.x / gridDim.x, u_end = U * (blockIdx.x + 1) / gridDim.x;
    const int per_z = d_m_tiles * d_n_ntiles;
    const uint32_t b_bytes = (uint32_t)d_nt * 128u;

    // item = 1 or 2 consecutive units (same split, same N tile, adjacent row tiles) sharing every weight tile
#define CH_FOR_ITEMS()                                                                                         \
    for (int64_t u = u_begin, _n; u < u_end; u += _n)                                                          \
      if (const int z = (int)(u / per_z), r_ = (int)(u - (int64_t)z * per_z), nti = r_ / d_m_tiles,            \
          m = r_ - nti * d_m_tiles, nsub = (d_nsub_max == 2 && u + 1 < u_end && m + 1 < d_m_tiles) ? 2 : 1,    \
          t_begin = min(z * d_sps, T), t_end = min(t_begin + d_sps, T);                                        \
          (_n = nsub, true))

    if (warp == CH_W_B) {
      // ============================ weight tiles ====================================
      const uint8_t *wtiles = s_desc->wtiles;
      CH_FOR_ITEMS() {
        (void)m;
        for (int t = t_begin; t < t_end; ++t) {
          mbar_wait_relaxed(emptyB + 8 * b_slot, b_phase ^ 1, 64);
          if (elect_one()) {
            const uint32_t fb = fullB + 8 * b_slot;
            if (flags & 0x200) {                      // tuning: no weight loads
              mbar_expect_tx(fb, 0u);
            } else {
              mbar_expect_tx(fb, b_bytes);
              bulk_g2s(b_ring_k + b_slot * (uint32_t)bslot, wtiles + ((int64_t)t * d_n_ntiles + nti) * b_bytes, b_bytes, fb);
            }
          }
          __syncwarp();
          if (++b_slot == (uint32_t)sb) { b_slot = 0; b_phase ^= 1; }
        }
      }
    } else if (warp < CH_W_MMA) {
      // ================= gathered A rows: warp w fills every CH_A_WARPS-th row slot, all 128 rows of it ====================
      // 8 lanes cover one 128-byte row line (one L2 line), 4 rows per copy instruction, 32 instructions per slot behind ONE
      // barrier wait and ONE (self-tracking) arrival; the destination carries the 128B swizzle (chunk ^ (row & 7)); a
      // missing neighbour is a zero-fill copy.  The slot's 128 row indices are four coalesced loads (lane l: rows l, l+32, ..)
      // fetched one slot of this warp ahead and handed round by shuffles.
      const int w = warp - CH_W_A, j = lane & 7, q = lane >> 3;
      const int32_t *nbr = s_desc->nbr;
      const uint8_t *src0 = s_desc->src0 + j * 16, *src1 = s_desc->src1 + j * 16;
      const uint32_t rb0 = (uint32_t)d_nb0 * 128u, rb1 = (uint32_t)d_nb1 * 128u;
      const uint32_t off_even = (uint32_t)q * 128u + (uint32_t)((j ^ q) << 4);                 // rows 8n + q
      const uint32_t off_odd = (uint32_t)(4 + q) * 128u + (uint32_t)((j ^ (4 + q)) << 4);      // rows 8n + 4 + q
      // Ring slot s is always filled by warp s % CH_A_WARPS, lap after lap: a warp cannot run a lap ahead of itself, so the
      // parity of a slot's empty barrier is unambiguous (with slots dealt round-robin over the warps, a fast warp one lap
      // ahead of a slow one passed the parity test early and overwrote rows that had not been multiplied yet).
      CH_FOR_ITEMS() {
        (void)nti;
        const uint32_t n_slots = (uint32_t)((t_end - t_begin) * nsub), g_end = g_slot + n_slots;
        auto decode = [&](uint32_t jl_, int &k_, int &cb_, int &s_) {
          const int st = (int)jl_ / nsub;             // stage-major, sub-tile-minor: the order the consumers take slots in
          s_ = (int)jl_ - st * nsub;
          const int tt = t_begin + st;
          k_ = tt / nb; cb_ = tt - k_ * nb;
        };
        auto fetch = [&](int k_, int s_, int32_t (&r)[4]) {
          const int32_t *nk = nbr ? nbr + (int64_t)k_ * d_n_out : nullptr;
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int64_t o = (int64_t)(m + s_) * CH_M + 32 * i + lane;
            r[i] = (o < d_n_out) ? (nk ? __ldg(nk + o) : (int32_t)o) : -1;
          }
        };
        int32_t nxt[4];
        int k_n = 0, cb_n = 0, s_n = 0;
        const bool owner = (uint32_t)w < (uint32_t)sa;
        if (owner && p_lapb + p_sl < g_end) { decode(p_lapb + p_sl - g_slot, k_n, cb_n, s_n); fetch(k_n, s_n, nxt); }
        while (owner && p_lapb + p_sl < g_end) {
          int32_t cur[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) cur[i] = nxt[i];
          const int cb = cb_n;
          const uint32_t sl = p_sl, par = p_par, jl = p_lapb + p_sl - g_slot;
          // my next slot (same warp, CH_A_WARPS slots on or the next lap)
          p_sl += CH_A_WARPS;
          if (p_sl >= (uint32_t)sa) { p_sl = (uint32_t)w; p_lapb += (uint32_t)sa; p_par ^= 1u; }
          if (p_lapb + p_sl < g_end) { decode(p_lapb + p_sl - g_slot, k_n, cb_n, s_n); fetch(k_n, s_n, nxt); }   // its row indices, ahead of time
          const bool first = cb < d_nb0;
          const uint8_t *src = (first ? src0 : src1) + (first ? cb : cb - d_nb0) * 128;
          const uint32_t rb = first ? rb0 : rb1;
          chain_wait(emptyA + 8 * sl, par ^ 1u, 4 | ((int)jl << 8));
          const uint32_t a_dst = a_ring_k + sl * (uint32_t)CH_A_BYTES;
          if (!(flags & 0x100)) {                     // tuning: bit 8 = no row copies
#pragma unroll
            for (int g8 = 0; g8 < 4; ++g8) {          // 8 copy instructions at a time: shuffles first, then the copies
              int32_t r8[8];
#pragma unroll
              for (int ii = 0; ii < 8; ++ii) r8[ii] = __shfl_sync(0xffffffffu, cur[g8], (4 * ii + q) & 31);   // rows 32 g8 + 4 ii + q
#pragma unroll
              for (int ii = 0; ii < 8; ++ii) {
                const int i = g8 * 8 + ii;
                const uint32_t rr = r8[ii] < 0 ? 0u : (uint32_t)r8[ii];
                // src-size form (16 or 0 bytes): the copy engine itself writes the zeros of a missing neighbour, so they are
                // covered by the self-tracking arrival below (zeros written by any other path would not be).
                cp_async16(a_dst + (uint32_t)(i >> 1) * 1024u + ((i & 1) ? off_odd : off_even), src + (uint64_t)rr * rb,
                           r8[ii] < 0 ? 0u : 16u);
              }
            }
          }
          cp_async_arrive_noinc(fullA + 8 * sl);      // 32 self-tracking arrivals, fired by the copy engine
        }
        g_slot = g_end;
      }
    } else {
      // ============ consumers: warpgroup g multiplies rows [64g, 64g+64) of every sub-tile of an item, then stores them ========
      // (chain_item, one instance per N-tile width and sub-tile count: two sub-tiles only with N tiles of at most 128 columns)
      const int g = (warp - CH_W_MMA) >> 2;
      const ChainRings R{a_ring_k, b_ring_k, (uint32_t)bslot, (uint32_t)sa, (uint32_t)sb, fullA, emptyA, fullB, emptyB};
      const uint32_t stgw = stg_u32 + (uint32_t)(warp - CH_W_MMA) * 2048u;
      const bool no_store = (flags & 0x800) != 0;
      const int nch = d_nt / 32;
      CH_FOR_ITEMS() {
#define CH_ITEM(n, s)                                                                                                  \
          case n: chain_item<n, s>(R, *s_desc, s_ss, stgw, no_store, a_slot, a_phase, b_slot, b_phase, t_begin, t_end, z, nti, \
                                   m, g, warp, lane); break;
        if (nsub == 2) {
          switch (nch) {
            CH_ITEM(1, 2) CH_ITEM(2, 2)
            default: __trap();                        // osb_conv_desc_fill pairs sub-tiles only for N tiles <= CH_MAX_PAIR_NT
          }
        } else {
          switch (nch) {
            CH_ITEM(1, 1) CH_ITEM(2, 1) CH_ITEM(3, 1) CH_ITEM(4, 1)
            default: __trap();                        // osb_conv_desc_fill plans N tiles of at most 128 columns
          }
        }
#undef CH_ITEM
      }
    }
#undef CH_FOR_ITEMS

    if (d_nsplit > 1) {
      // ---- split-K: every partial is in global memory after this barrier; reduce + epilogue by all threads of the grid
      grid_barrier(gbar, bar_gen);
      const ConvDesc &d = args.d[L];
      const int groups = d.cout / 8;
      const int64_t total = d.n_out * groups;
      for (int64_t e = (int64_t)blockIdx.x * CH_THREADS + tid; e < total; e += (int64_t)gridDim.x * CH_THREADS) {
        const int64_t o = e / groups;
        const int c0 = (int)(e - o * groups) * 8;
        float y[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int z = 0; z < d.nsplit; ++z) {
          const float4 *pp = reinterpret_cast<const float4 *>(d.partial + ((int64_t)z * d.n_out + o) * d.cout_pad + c0);
          const float4 a = __ldcg(pp), b = __ldcg(pp + 1);
          y[0] += a.x; y[1] += a.y; y[2] += a.z; y[3] += a.w; y[4] += b.x; y[5] += b.y; y[6] += b.z; y[7] += b.w;
        }
        if (d.scale) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) y[jj] = fmaf(y[jj], s_ss[c0 + jj], s_ss[CH_SS_FLOATS + c0 + jj]);
        }
        const int64_t off = o * (int64_t)d.cout * 4 + split_off_hi(c0);
        if (d.res) {
          const uint4 hq = __ldcg(reinterpret_cast<const uint4 *>(d.res + off)), lq = __ldcg(reinterpret_cast<const uint4 *>(d.res + off + 64));
          const __nv_bfloat16 *hh = reinterpret_cast<const __nv_bfloat16 *>(&hq);
          const __nv_bfloat16 *ll = reinterpret_cast<const __nv_bfloat16 *>(&lq);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) y[jj] += join_bf16(hh[jj], ll[jj]);
        }
        if (d.relu) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) y[jj] = fmaxf(y[jj], 0.f);
        }
        if (d.out_split) {
          __align__(16) __nv_bfloat16 hh[8], ll[8];
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) split_bf16(y[jj], hh[jj], ll[jj]);
          *reinterpret_cast<uint4 *>(d.out_split + off) = *reinterpret_cast<const uint4 *>(hh);
          *reinterpret_cast<uint4 *>(d.out_split + off + 64) = *reinterpret_cast<const uint4 *>(ll);
        }
        if (d.out_f32) {
          const int64_t orow = d.out_row_map ? (int64_t)__ldg(d.out_row_map + o) : o;
          float4 *op = reinterpret_cast<float4 *>(d.out_f32 + orow * d.cout + c0);
          op[0] = make_float4(y[0], y[1], y[2], y[3]);
          op[1] = make_float4(y[4], y[5], y[6], y[7]);
        }
      }
    }
  }

  if (dbg_clock && tid == 0) dbg_clock[blockIdx.x * 32 + 2] = clock64();
}

// ------------------------------------------------------------ tile-major, pre-swizzled weight packing
// wtiles[((k*nb + cb) * n_ntiles + nti)] = nt rows (output channels) x 128 B, each row the split line
// [hi ch0-15 | hi ch16-31 | lo ch0-15 | lo ch16-31] of input channels [32cb, 32cb+32), with the 16-byte chunks of row n
// stored at chunk ^ (n & 7): exactly what a 128B-swizzled TMA tile load would leave in shared memory, so that one
// linear cp.async.bulk per stage fetches a ready-to-multiply B operand (no tensor map, nothing to encode per launch).
__global__ void k_pack_weight_tiles(const float *__restrict__ w, int K, int cin, int cout, int cout_pad, int nt, int transpose_w,
                                    uint8_t *__restrict__ wt) {
  const int nb = cin / 32, n_ntiles = cout_pad / nt;
  const int64_t total = (int64_t)K * cout_pad * cin;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(e % cin);
    const int64_t kn = e / cin;
    const int ng = (int)(kn % cout_pad), k = (int)(kn / cout_pad);
    float v = 0.f;
    if (ng < cout) v = transpose_w ? w[((int64_t)k * cout + ng) * cin + c] : w[((int64_t)k * cin + c) * cout + ng];
    __nv_bfloat16 hi, lo;
    split_bf16(v, hi, lo);
    const int cb = c >> 5, ci = c & 31, nti = ng / nt, n = ng - nti * nt;
    uint8_t *tile = wt + ((((int64_t)k * nb + cb) * n_ntiles) + nti) * (int64_t)nt * 128;
    const int jh = ci >> 3, el = ci & 7;
    *reinterpret_cast<__nv_bfloat16 *>(tile + n * 128 + (((jh) ^ (n & 7)) << 4) + el * 2) = hi;
    *reinterpret_cast<__nv_bfloat16 *>(tile + n * 128 + (((4 + jh) ^ (n & 7)) << 4) + el * 2) = lo;
  }
}

}  // namespace osb

namespace osb { bool conv_tc_tuning(const char *name, int64_t v); }
using namespace osb;

// Tile shapes keep a consumer thread at most 64 fp32 accumulators ((64 rows x N columns) / 128 threads per sub-tile), which
// fit its registers beside the kernel's persistent state with no spill: N tiles of at most 128 columns, and two sub-tiles
// per item only for N tiles of at most 64 columns (CH_MAX_PAIR_NT).  Wider outputs are padded to whole 128-column tiles.
static inline int chain_cout_pad(int cout) { return cout <= 128 ? (cout + 15) / 16 * 16 : (cout + 127) / 128 * 128; }
static inline int chain_nt(int cout) { const int cp = chain_cout_pad(cout); return cp <= 128 ? cp : 128; }
constexpr int CH_MAX_PAIR_NT = 64;

extern "C" {

size_t osb_conv_desc_bytes(void) { return sizeof(ConvDesc); }

size_t osb_conv_weight_tiles_bytes(int32_t K, int32_t cin, int32_t cout) { return (size_t)K * chain_cout_pad(cout) * cin * 4; }

int osb_conv_pack_weight_tiles(const float *w, int32_t K, int32_t cin, int32_t cout, int32_t transpose_w, void *wtiles, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(K >= 1 && cin % 32 == 0 && cin > 0 && cout > 0, "osb_conv_pack_weight_tiles: cin (%d) must be a multiple of 32", cin);
  const int cp = chain_cout_pad(cout), nt = chain_nt(cout);
  const int64_t total = (int64_t)K * cp * cin;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(total, 256), 132 * 32);
  k_pack_weight_tiles<<<grid, 256, 0, stream>>>(w, K, cin, cout, cp, nt, transpose_w, (uint8_t *)wtiles);
  OSB_LAUNCH_CHECK();
  return 0;
}

// Split factor of one layer when it runs on a grid of `grid_ctas` CTAs.  Base rule: as many splits as it takes to give every
// CTA a unit (grid / tiles).  That rule leaves half of the SMs idle on 76-tile levels (9.7 k rows: one unit of 108 stages per
// busy CTA), so a small cost model may RAISE the factor when it predicts a clear gain (it never lowers it: for the smallest
// levels the measured optimum is the base rule):
//   main loop   per CTA (pairs of units x ~0.75 us + single units x ~0.6 us) x stages per split; an item is two row-adjacent
//               units when the N tile is <= CH_MAX_PAIR_NT wide; 1.6x for wider N tiles
//   split cost  ~10 us (grid barrier, partial tiles out, reduce pass) + the partials written and read once at ~5 TB/s (L2)
// The constants are rough per-stage costs of the bench scene's layers; the rules above (never lower than the base rule,
// a clear predicted gain to raise it) keep a mis-fitted constant from doing harm.
static int chain_nsplit(int64_t n_out, int K, int cin, int cout, int grid_ctas, int force, int nsub_knob) {
  const int cp = chain_cout_pad(cout), nt = chain_nt(cout);
  const int64_t tiles = ceil_div(n_out, CH_M) * (cp / nt);
  const int T = K * (cin / 32);
  const int cap = std::max(1, std::min(32, T));
  if (force > 0) return std::min(force, cap);
  const bool pairs = nt <= CH_MAX_PAIR_NT && nsub_knob >= 2;
  const int base = (int)std::max<int64_t>(1, std::min<int64_t>(grid_ctas / tiles, cap));
  auto cost = [&](int ns, bool &ok) {
    const int sps = (T + ns - 1) / ns;
    ok = (T + sps - 1) / sps == ns;                                // else this many splits would leave empty ones
    const int64_t upc = ceil_div(tiles * ns, (int64_t)grid_ctas);
    const double per = pairs ? (double)(upc / 2) * 0.75 + (double)(upc % 2) * 0.6 : (double)upc * 0.6 * 1.6;
    double us = per * sps + 4.0;
    if (ns > 1) {
      const double partial_bytes = (double)ns * (double)n_out * cp * 4.0;
      if (partial_bytes > 64e6) ok = false;                        // scratch stays small (the engine provides 96 MB per layer)
      us += 10.0 + 2.0 * partial_bytes / 5e6;
    }
    return us;
  };
  bool ok = true;
  double best = cost(base, ok);
  int best_ns = base;
  for (int ns = base + 1; ns <= cap; ++ns) {
    const double us = cost(ns, ok);
    if (ok && us < best - std::max(0.5, 0.08 * best)) { best = us; best_ns = ns; }
  }
  return best_ns;
}

static int g_chain_force_split = 0;      // tuning: > 0 forces the split factor of every layer (1 disables splitting)
static int g_chain_nsub = 2;             // tuning: 1 = never pair sub-tiles
static int g_chain_grid = 0;             // tuning: CTAs per launch (0 = one per SM)
static int g_chain_sa = 0, g_chain_sb = 0;   // tuning: ring depths (0 = as many row slots as fit / 3 or 2 weight slots)
static long long *g_chain_dbg_clock = nullptr;
static int g_chain_dbg_skip = 0;         // tuning: bit0 no row copies, bit1 no weight loads, bit3 no stores

int osb_tuning_set(const char *name, int64_t value) {
  const std::string n(name ? name : "");
  if (n == "chain_force_split") g_chain_force_split = (int)value;
  else if (n == "chain_nsub") g_chain_nsub = (int)value;
  else if (n == "chain_grid") g_chain_grid = (int)value;
  else if (n == "chain_sa") g_chain_sa = (int)value;
  else if (n == "chain_sb") g_chain_sb = (int)value;
  else if (n == "chain_dbg_clock") g_chain_dbg_clock = (long long *)(intptr_t)value;
  else if (n == "chain_dbg_skip") g_chain_dbg_skip = (int)value;
  else if (n == "chain_report") {               // host-mapped int64 buffer [1 + 4*1024]: where a stuck wait was (tuning)
    long long *ptr = (long long *)(intptr_t)value;
    OSB_CUDA(cudaMemcpyToSymbol(g_chain_report, &ptr, sizeof(ptr)));
  }
  else { OSB_CHECK(conv_tc_tuning(n.c_str(), value), "osb_tuning_set: unknown knob '%s'", n.c_str()); }
  return 0;
}

int osb_conv_chain_grid(void) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // the grid barrier needs every CTA resident at once: one CTA per SM at most
  return g_chain_grid > 0 ? std::min(g_chain_grid, sms) : sms;
}

size_t osb_conv_chain_workspace_bytes(int64_t n_out, int32_t K, int32_t cin, int32_t cout) {
  if (n_out <= 0 || K < 1 || cin < 32 || cout <= 0) return 0;     // shapes osb_conv_desc_fill rejects: nothing to reserve
  const int ns = chain_nsplit(n_out, K, cin, cout, osb_conv_chain_grid(), g_chain_force_split, g_chain_nsub);
  return ns > 1 ? (size_t)ns * n_out * chain_cout_pad(cout) * sizeof(float) : 0;
}

int osb_conv_desc_fill(void *desc_host, const void *src0, int32_t c0, const void *src1, int32_t c1, const int32_t *nbr, int64_t n_out,
                       int32_t K, const void *wtiles, int32_t cout, const float *scale, const float *shift, const void *res,
                       int32_t relu, void *out_split, float *out_f32, const int32_t *out_row_map, const int32_t *cmap,
                       int32_t cmap_cout, void *ws, size_t ws_bytes, int32_t barrier_before) {
  OSB_CHECK(desc_host != nullptr, "osb_conv_desc_fill: no descriptor");
  OSB_CHECK(src0 && c0 > 0 && c0 % 32 == 0 && c1 >= 0 && c1 % 32 == 0, "osb_conv_desc_fill: channel counts must be multiples of 32 (c0=%d c1=%d)", c0, c1);
  OSB_CHECK((c1 == 0) == (src1 == nullptr), "osb_conv_desc_fill: src1 / c1 mismatch");
  OSB_CHECK(K >= 1 && K <= 32, "osb_conv_desc_fill: K=%d not supported (<= 32)", K);
  OSB_CHECK(nbr != nullptr || K == 1, "osb_conv_desc_fill: identity map needs K == 1");
  OSB_CHECK(n_out > 0 && n_out < (1ll << 31), "osb_conv_desc_fill: bad row count");
  OSB_CHECK(cout % 32 == 0 && cout > 0, "osb_conv_desc_fill: cout (%d) must be a multiple of 32", cout);
  OSB_CHECK(out_split || out_f32, "osb_conv_desc_fill: no output given");
  OSB_CHECK((scale == nullptr) == (shift == nullptr), "osb_conv_desc_fill: scale and shift go together");
  OSB_CHECK(cmap == nullptr || (cmap_cout > 0 && cmap_cout % 32 == 0 && cout % cmap_cout == 0 && res == nullptr),
            "osb_conv_desc_fill: bad dense-transpose arguments");
  OSB_CHECK((cmap ? cmap_cout : cout) <= CH_SS_FLOATS, "osb_conv_desc_fill: more than %d output channels per row", CH_SS_FLOATS);
  ConvDesc d{};
  const int cin = c0 + c1;
  d.src0 = (const uint8_t *)src0; d.src1 = (const uint8_t *)src1; d.nbr = nbr; d.wtiles = (const uint8_t *)wtiles;
  d.scale = scale; d.shift = shift; d.res = (const uint8_t *)res; d.out_split = (uint8_t *)out_split; d.out_f32 = out_f32;
  d.out_row_map = out_row_map; d.cmap = cmap; d.n_out = n_out; d.K = K; d.nb0 = c0 / 32; d.nb1 = c1 / 32;
  d.cout = cout; d.cout_pad = chain_cout_pad(cout); d.nt = chain_nt(cout); d.n_ntiles = d.cout_pad / d.nt;
  d.relu = relu; d.cmap_cout = cmap_cout; d.m_tiles = (int)ceil_div(n_out, CH_M);
  d.nsub_max = (d.nt <= CH_MAX_PAIR_NT && g_chain_nsub >= 2) ? 2 : 1;
  d.barrier_before = barrier_before ? 1 : 0;
  d.nsplit = cmap ? 1 : chain_nsplit(n_out, K, cin, cout, osb_conv_chain_grid(), g_chain_force_split, g_chain_nsub);
  const int T = K * (cin / 32);
  d.stages_per_split = (T + d.nsplit - 1) / d.nsplit;
  d.nsplit = (T + d.stages_per_split - 1) / d.stages_per_split;            // no empty splits
  d.partial = nullptr;
  if (d.nsplit > 1) {
    const size_t need = (size_t)d.nsplit * n_out * d.cout_pad * sizeof(float);
    OSB_CHECK(ws != nullptr && ws_bytes >= need, "osb_conv_desc_fill: workspace of %zu bytes required (got %zu)", need, ws_bytes);
    d.partial = (float *)ws;
  }
  memcpy(desc_host, &d, sizeof(d));
  return 0;
}

int osb_conv_chain_launch(const void *descs_host, int32_t n_layers, void *grid_barrier_dev, int32_t flags, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(descs_host && n_layers >= 1, "osb_conv_chain_launch: bad arguments");
  const ConvDesc *h = (const ConvDesc *)descs_host;
  for (int i = 0; i < n_layers; ++i) {
    OSB_CHECK(i > 0 || !h[i].barrier_before, "osb_conv_chain_launch: the first layer of a launch cannot ask for a barrier");
    // a split layer's reduce phase is not followed by a barrier: the next layer may only reuse the partial buffer behind one
    OSB_CHECK(i == 0 || h[i].barrier_before || h[i].nsplit == 1 || h[i - 1].nsplit == 1 || h[i].partial != h[i - 1].partial,
              "osb_conv_chain_launch: layers %d and %d share a split workspace without a barrier between them", i - 1, i);
  }
  OSB_SMEM_ATTR_ONCE(k_conv_chain, 227 * 1024);
  const int grid = osb_conv_chain_grid();
  // the layer descriptors travel as kernel parameters: at most CH_MAX_LAYERS per launch, longer lists in several launches
  // (a launch boundary orders everything, so the first layer of a later launch needs no grid barrier)
  for (int l0 = 0; l0 < n_layers; l0 += CH_MAX_LAYERS) {
    const int cnt = std::min(CH_MAX_LAYERS, n_layers - l0);
    ChainArgs args;
    memcpy(args.d, h + l0, sizeof(ConvDesc) * cnt);
    args.d[0].barrier_before = 0;
    int nt_max = 0, need_bar = 0;
    for (int i = 0; i < cnt; ++i) {
      nt_max = std::max(nt_max, args.d[i].nt);
      need_bar |= (args.d[i].barrier_before || args.d[i].nsplit > 1);
    }
    OSB_CHECK(!need_bar || grid_barrier_dev != nullptr, "osb_conv_chain_launch: this chain needs the grid-barrier words");
    const int bslot = nt_max * 128;
    const int fixed = 1024 + CH_STG_BYTES + 2 * CH_SS_FLOATS * 4 + 40 * 8 + 64;   // alignment slack, staging, BN constants, barriers
    int sb = g_chain_sb > 0 ? g_chain_sb : (bslot >= 32768 ? 2 : 3);
    sb = std::min(sb, CH_MAX_SB);
    int sa = (227 * 1024 - fixed - sb * bslot) / CH_A_BYTES;
    if (g_chain_sa > 0) sa = std::min(sa, g_chain_sa);
    sa = std::min(sa, CH_MAX_SA);
    // An EVEN ring: the two row slots of a paired stage then never straddle the end of the ring, and these are the ring
    // shapes tests/test_chain_protocol_model.py proves safe and live.  At least four slots: a consumer warpgroup holds the
    // row slots of two paired stages at once (it releases a stage's slots once the next stage's wgmmas are issued and the
    // previous group has retired).
    sa &= ~1;
    OSB_CHECK(sa >= 4, "osb_conv_chain_launch: shared memory does not hold four row slots");
    const size_t smem_bytes = (size_t)sa * CH_A_BYTES + (size_t)sb * bslot + fixed;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(CH_THREADS); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cfg.attrs = attr; cfg.numAttrs = (flags & 1) ? 1 : 0;
    OSB_CUDA(cudaLaunchKernelEx(&cfg, k_conv_chain, args, (int)cnt, (unsigned *)grid_barrier_dev, sa, sb, bslot,
                                (int)((flags & 1) | (g_chain_dbg_skip << 8)), g_chain_dbg_clock));
    OSB_LAUNCH_CHECK();
  }
  return 0;
}

}  // extern "C"
