// Open-vocabulary matching on tensor cores (wgmma) (run/evaluate.py:288-323).
//
//   scores[p, k] = fp16( sum_c a[p, c] * text[k, c] ),  a[p,:] = fp16( prep(feat[v(p), :]) ),  fp32 accumulation
//
// with prep = identity (`.half()`), or x / (|x| + 1e-5) (the normalised products of the ensemble branch), v(p) =
// inds_reverse[p] (voxel -> point expansion without materialising predictions[inds_reverse]), or a per-point choice
// between the 3-D and the fused 2-D feature (ensemble select).  The operands are rounded to fp16 exactly where the
// reference rounds them, so the [N_pts, C] x [C, K] product is the reference's own fp16 GEMM.
//
// One CTA = 128 points.  Warps 0-15 build the A operand: one warp per row at a time, the row lives in registers
// (coalesced 256-byte loads), is reduced for the norm, rounded to fp16 and written into the K-major 128B-swizzled
// shared-memory tile of all C/64 depth chunks (192 KB for C = 768).  Warp 16 streams the text matrix chunk by chunk with
// TMA (rows >= K_text are out of bounds -> zero fill).  Warps 0-7 (two warpgroups, 64 points each) then run `wgmma` f16
// (M=64, N=96 per pass, K=16) into register accumulators, round to fp16, keep the first-maximum argmax over the passes and
// write scores / labels / row maxima.  HBM-bound: 4*C (or 2*C) bytes per point against 2*C*K flops.
//
// k_match_tc_vote is the same kernel with the test-time repeat vote in the epilogue: each fp16 score is added into the
// caller's fp16 store in place and the labels of the score row and of the summed row are kept (vote.cuh), so a repeat's
// [N_pts, K] scores never reach HBM.  k_match_tc itself compiles to the same instructions as before the vote existed.
//
// k_match_tc_ce is the same kernel with the validation tail of run/distill.py in the epilogue (MatchTcCe below): the
// cross-entropy term, the argmax and the intersection / union / target counts of every row.  k_match_tc and
// k_match_tc_vote compile to the same instructions as before it existed.
//
// k_match_tc_topk is the same kernel with a running per-point top-k (k <= 8) in the epilogue (MatchTcTopk below), so the
// number of passes has no bound of its own: the result is [N_pts, k], never [N_pts, K].  The three kernels above compile
// to the same instructions as before it existed.  k_match_tc_topk<NP, true> takes its A tile from the FP8 scene index
// (mt_fill_a8: e4m3 codes and per-row exponents, the tile mt_fill_a writes for the rows d), which labels the index
// (search.py, SceneIndex.label) with the bits the fp16 kernel gives on d.
#include "match_tc.cuh"
#include "metric.cuh"
#include "vote.cuh"
#include <algorithm>

namespace osb {

// Test-time repeat vote (k_match_tc_vote): store[p,k] = fp16_rn(store[p,k] + scores[p,k]) in place, and the labels of
// this repeat's scores and of the accumulated sum (vote.cuh: torch CPU `max(1)[1]`, NaN-first).
struct MatchTcVote {
  __half *store;                     // [n_pts, k_text]
  int64_t *label_cur;                // [n_pts] or NULL
  int64_t *label_acc;                // [n_pts] or NULL
  int pair;                          // K even and the store 4-byte aligned: a thread's column pair is one __half2
};

// Validation cross-entropy (k_match_tc_ce, run/distill.py:419-431): per point row with label y, torch's CUDA log_softmax
// for Half read at y, logp = fp16((s_y - m) - log(sum_k exp(s_k - m))) in fp32, from a running (m, sum) per row over the
// 96-row passes; the NLL term -logp summed in fp64 (per-block partials, merged in block order by k_match_ce_loss), the
// NaN-first argmax (vote.cuh) and util.py's intersection / union / target counts (metric.cuh).  A label outside [0, K)
// other than ignore drops the row from the loss and the counts and is counted in *bad.
struct MatchTcCe {
  const void *label;                 // [n_pts] int32 or int64
  int label_is_i64, ignore, classes;
  double *part;                      // [gridDim.x][2]: sum of the terms, labelled rows
  unsigned long long *areas;         // [3, classes], accumulated
  int32_t *bad;                      // [1], accumulated
  void *loss;                        // fp16 [1]: fp16(sum / rows), written by k_match_ce_loss
};

// Streaming top-k (k_match_tc_topk): per point, the k best of all K fp16 scores, best first.  NaN ranks above every
// number (NaNs by ascending column), numbers by descending value with -0 == +0, equal values by ascending column; k = 1
// is vote.cuh's rule.  Each row keeps its list of k order keys (topk_key) in shared memory; a column is tested against
// the upper half of the row's k-th key, read once per pass, and only the columns that pass are offered to the list, one
// lane of the row's quad at a time.
struct MatchTcTopk {
  int k;                             // 1..8, at most K
  __half *scores;                    // [n_pts, k] or NULL
  int64_t *label;                    // [n_pts, k]
  const int8_t *row_exp;             // [n_pts] (k_match_tc_topk<NP, true>): p.feat holds e4m3 codes [n_pts, C]
};
constexpr int MT_TOPK_MAX = 8;

enum { MT_PLAIN = 0, MT_VOTE = 1, MT_CE = 2, MT_TOPK = 3 };

// the label of point row pt as an int: y in [0, K), ignore, or (a label outside [0, K)) a negative value other than ignore
__device__ __forceinline__ int ce_label(const MatchTcCe &ce, int64_t pt, int64_t n_pts, int k_text) {
  if (pt >= n_pts) return ce.ignore;
  const long long y = ce.label_is_i64 ? (long long)__ldg(reinterpret_cast<const int64_t *>(ce.label) + pt)
                                      : (long long)__ldg(reinterpret_cast<const int32_t *>(ce.label) + pt);
  if (y == ce.ignore || (y >= 0 && y < k_text)) return (int)y;
  return ce.ignore == -1 ? -2 : -1;
}

template <int NP, int MODE, bool F8 = false>   // half2 pairs per lane: C = 64 * NP
__device__ __forceinline__ void match_tc_body(const CUtensorMap &tmT, const MatchTcParams p, const MatchTcVote vo,
                                              const MatchTcCe ce, const MatchTcTopk tk) {
  constexpr bool VOTE = MODE == MT_VOTE, CE = MODE == MT_CE, TOPK = MODE == MT_TOPK;
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int C = 64 * NP;
  constexpr int A_BYTES = NP * MT_M * 128;                      // NP chunks of [128 rows x 128 B]
  constexpr int B_BYTES = MT_NW * 128;
  uint8_t *sA = smem, *sB = smem + A_BYTES;
  uint64_t *bars = reinterpret_cast<uint64_t *>(sB + MT_BSTAGES * B_BYTES);   // b_full[2], b_empty[2], a_full

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t row0 = (int64_t)blockIdx.x * MT_M;
  const uint32_t b_full = smem_u32(bars), b_empty = smem_u32(bars + 2), a_full = smem_u32(bars + 4);

  if (tid == 0) {
    // b_empty: one arrival per consumer warpgroup
    for (int s = 0; s < MT_BSTAGES; ++s) { mbar_init(b_full + 8 * s, 1); mbar_init(b_empty + 8 * s, 2); }
    mbar_init(a_full, MT_PW * 32);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (tid == MT_PW * 32) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmT) : "memory");
  // CE: the block's 128 NLL terms and labelled-row flags, then its [3, classes] histogram
  float *s_term = reinterpret_cast<float *>(sB + MT_BSTAGES * B_BYTES + 128);
  int *s_lab = reinterpret_cast<int *>(s_term + MT_M);
  uint32_t *s_hist = reinterpret_cast<uint32_t *>(s_lab + MT_M);
  // TOPK: the block's 128 lists of MT_TOPK_MAX order keys
  uint64_t *s_topk = reinterpret_cast<uint64_t *>(sB + MT_BSTAGES * B_BYTES + 128);
  if constexpr (CE)
    for (int b = tid; b < 3 * ce.classes; b += MT_THREADS) s_hist[b] = 0;
  __syncthreads();
  const int n_stage = p.n_pass * NP;

  if (warp < MT_PW) {
    // ============================ A producers: 8 rows per warp ==============================
    if constexpr (F8)
      mt_fill_a8<NP>(reinterpret_cast<const uint8_t *>(p.feat), tk.row_exp, p.n_pts, sA, row0, warp, lane);
    else
      mt_fill_a<NP>(p, sA, row0, warp, lane);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");           // generic-proxy writes -> wgmma reads
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(a_full) : "memory");
  } else if (warp == MT_PW) {
    // ============================ TMA producer: text chunks ==================================
    int s = 0; uint32_t phase = 0;
    for (int t = 0; t < n_stage; ++t) {
      const int pass = t / NP, c = t % NP;
      mbar_wait(b_empty + 8 * s, phase ^ 1);
      if (elect_one()) {
        mbar_expect_tx(b_full + 8 * s, (uint32_t)B_BYTES);
        tma_load_2d(smem_u32(sB + s * B_BYTES), &tmT, b_full + 8 * s, c * 64, pass * MT_NW);
      }
      __syncwarp();
      if (++s == MT_BSTAGES) { s = 0; phase ^= 1; }
    }
  }

  if (warp < 8) {
    // ============ wgmma: warpgroup g multiplies points [64g, 64g + 64), pass by pass; fp16 rounding, argmax ============
    const int g = warp >> 2;
    const int r_lo = 64 * g + 16 * (warp & 3) + (lane >> 2);      // this thread's rows: r_lo and r_lo + 8
    const int cq = 2 * (lane & 3);
    float best[2] = {-INFINITY, -INFINITY};
    int best_k[2] = {0, 0};
    VoteArgmax vcur[2], vacc[2];
    if constexpr (VOTE) { vcur[0].init(); vcur[1].init(); vacc[0].init(); vacc[1].init(); }
    // CE: running max / sum of exp(s - max) over this thread's columns, and the label's score (the label is re-read
    // from L1 in every epilogue rather than held in registers across the products)
    float lm[2], ls[2], sy[2];
    if constexpr (CE) {
#pragma unroll
      for (int h = 0; h < 2; ++h) { lm[h] = -INFINITY; ls[h] = 0.f; sy[h] = 0.f; vcur[h].init(); }
    }
    if constexpr (TOPK) {   // empty lists: key 0 is below every valid key
#pragma unroll
      for (int h = 0; h < 2; ++h)
        for (int j = lane & 3; j < MT_TOPK_MAX; j += 4) s_topk[(r_lo + 8 * h) * MT_TOPK_MAX + j] = 0;
      __syncwarp();
    }
    mbar_wait(a_full, 0);
    int s = 0; uint32_t phase = 0;
    for (int pass = 0; pass < p.n_pass; ++pass) {
      float acc[MT_NW / 2];
#pragma unroll
      for (int i = 0; i < MT_NW / 2; ++i) acc[i] = 0.f;
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
      // CE, TOPK: this pass's fp16 scores of both rows as half2 pairs (the accumulators die here)
      __half2 hs[2][MT_NW / 8];
      if constexpr (CE || TOPK) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < MT_NW / 8; ++i) hs[h][i] = __floats2half2_rn(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t pt = row0 + r_lo + 8 * h;
        // CE: the label, then per column the score, the argmax, the pass maximum and the label's score
        int y = 0;
        float pm = -INFINITY;
        if constexpr (CE) y = ce_label(ce, pt, p.n_pts, p.k_text);
        // TOPK: the row's k-th key, and the columns of this thread that beat it
        uint64_t *row_topk = s_topk + (r_lo + 8 * h) * MT_TOPK_MAX;
        uint32_t thr = 0, cand = 0;
        if constexpr (TOPK) thr = (uint32_t)(row_topk[tk.k - 1] >> 32);
#pragma unroll
        for (int i = 0; i < MT_NW / 8; ++i) {
          if constexpr (VOTE) {
            // the thread's two adjacent columns k0, k0 + 1 of this row (k0 even): one 4-byte store access when the pair is
            // aligned (vo.pair), two 2-byte accesses otherwise
            const int k0 = pass * MT_NW + 8 * i + cq;
            if (k0 < p.k_text) {
              const bool two = k0 + 1 < p.k_text;
              const __half h0 = __float2half_rn(acc[4 * i + 2 * h]);
              const __half h1 = __float2half_rn(acc[4 * i + 2 * h + 1]);
              if (p.scores != nullptr && pt < p.n_pts) {
                p.scores[pt * p.k_text + k0] = h0;
                if (two) p.scores[pt * p.k_text + k0 + 1] = h1;
              }
              vcur[h].take(__half2float(h0), k0);
              if (two) vcur[h].take(__half2float(h1), k0 + 1);
              if (pt < p.n_pts) {
                __half *st = vo.store + pt * p.k_text + k0;
                __half s0, s1;
                if (two && vo.pair) {
                  // one fp16 add per lane, round to nearest even
                  const __half2 sum = __hadd2(*reinterpret_cast<const __half2 *>(st), __halves2half2(h0, h1));
                  *reinterpret_cast<__half2 *>(st) = sum;
                  s0 = __low2half(sum);
                  s1 = __high2half(sum);
                } else {
                  s0 = __hadd(st[0], h0);
                  st[0] = s0;
                  s1 = s0;
                  if (two) { s1 = __hadd(st[1], h1); st[1] = s1; }
                }
                vacc[h].take(__half2float(s0), k0);
                if (two) vacc[h].take(__half2float(s1), k0 + 1);
              }
            }
          } else if constexpr (CE) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int k = pass * MT_NW + 8 * i + cq + e;
              if (k < p.k_text) {
                const __half hv = e ? __high2half(hs[h][i]) : __low2half(hs[h][i]);
                const float sc = __half2float(hv);
                if (p.scores != nullptr && pt < p.n_pts) p.scores[pt * p.k_text + k] = hv;
                vcur[h].take(sc, k);
                pm = fmaxf(pm, sc);
                if (k == y) sy[h] = sc;
              }
            }
          } else if constexpr (TOPK) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int k = pass * MT_NW + 8 * i + cq + e;
              if (k < p.k_text) {
                const __half hv = e ? __high2half(hs[h][i]) : __low2half(hs[h][i]);
                const float sc = __half2float(hv);
                if (sc > best[h]) { best[h] = sc; best_k[h] = k; }   // smax: the rule of the plain kernel
                if ((uint32_t)(topk_key(hv, k) >> 32) >= thr) cand |= 1u << (2 * i + e);   // a superset of the survivors
              }
            }
          } else {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int k = pass * MT_NW + 8 * i + cq + e;       // ascending per thread: the first maximum is kept
              if (k < p.k_text) {
                const __half hv = __float2half_rn(acc[4 * i + 2 * h + e]);
                const float sc = __half2float(hv);
                if (p.scores != nullptr && pt < p.n_pts) p.scores[pt * p.k_text + k] = hv;
                if (sc > best[h]) { best[h] = sc; best_k[h] = k; }
              }
            }
          }
        }
        if constexpr (CE) {   // the pass's exp sum against the new running maximum
          const float mn = fmaxf(lm[h], pm), mu = mn == -INFINITY ? 0.f : mn;
          float sum = ls[h] * expf(lm[h] - mu);
#pragma unroll
          for (int i = 0; i < MT_NW / 8; ++i) {
            const float2 f = __half22float2(hs[h][i]);
            const int k = pass * MT_NW + 8 * i + cq;
            if (k < p.k_text) sum += expf(f.x - mu);
            if (k + 1 < p.k_text) sum += expf(f.y - mu);
          }
          lm[h] = mn; ls[h] = sum;
        }
        if constexpr (TOPK) {   // the survivors, one lane of each quad at a time (rare once the lists are full)
          if (__any_sync(0xffffffffu, cand != 0)) {
#pragma unroll 1
            for (int q = 0; q < 4; ++q) {
              if ((lane & 3) == q && cand != 0) {
#pragma unroll
                for (int i = 0; i < MT_NW / 8; ++i)
#pragma unroll
                  for (int e = 0; e < 2; ++e)
                    if ((cand >> (2 * i + e)) & 1u)
                      topk_insert(row_topk, tk.k,
                                  topk_key(e ? __high2half(hs[h][i]) : __low2half(hs[h][i]), pass * MT_NW + 8 * i + cq + e));
              }
              __syncwarp();
            }
          }
        }
      }
    }
    if constexpr (VOTE) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        vcur[h].reduce<4>();
        vacc[h].reduce<4>();
        const int64_t pt = row0 + r_lo + 8 * h;
        if ((lane & 3) == 0 && pt < p.n_pts) {
          if (vo.label_cur) vo.label_cur[pt] = vcur[h].k;
          if (vo.label_acc) vo.label_acc[pt] = vacc[h].k;
        }
      }
    } else if constexpr (CE) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        vcur[h].reduce<4>();
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {   // merge (max, sum) over the four lanes of the row
          const float om = __shfl_xor_sync(0xffffffffu, lm[h], o), os = __shfl_xor_sync(0xffffffffu, ls[h], o);
          const float mn = fmaxf(lm[h], om), mu = mn == -INFINITY ? 0.f : mn;
          ls[h] = ls[h] * expf(lm[h] - mu) + os * expf(om - mu);
          lm[h] = mn;
        }
        const int r = r_lo + 8 * h;
        const int64_t pt = row0 + r;
        const int y = ce_label(ce, pt, p.n_pts, p.k_text);
        // column y belongs to lane (y % 8) / 2 of the row's quad (96 % 8 == 0)
        const bool in_k = y >= 0 && y < p.k_text;
        const float s_y = __shfl_sync(0xffffffffu, sy[h], (lane & ~3) | (in_k ? (y & 7) >> 1 : 0));
        if ((lane & 3) == 0) {
          const bool live = pt < p.n_pts, lab = live && y != ce.ignore, bad = lab && !in_k;
          s_lab[r] = lab && in_k;
          s_term[r] = lab && in_k ? -__half2float(__float2half_rn((s_y - lm[h]) - logf(ls[h]))) : 0.f;
          if (bad) atomicAdd(ce.bad, 1);
          else if (live) inter_union_add(vcur[h].k, y, ce.classes, ce.ignore, s_hist);
          if (live && p.label) p.label[pt] = vcur[h].k;
        }
      }
    } else if constexpr (TOPK) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {   // smax as the plain kernel merges it
          const float ob = __shfl_xor_sync(0xffffffffu, best[h], o);
          const int ok = __shfl_xor_sync(0xffffffffu, best_k[h], o);
          if (ob > best[h] || (ob == best[h] && ok < best_k[h])) { best[h] = ob; best_k[h] = ok; }
        }
        const int r = r_lo + 8 * h;
        const int64_t pt = row0 + r;
        if (pt < p.n_pts) {
          for (int j = lane & 3; j < tk.k; j += 4) {
            const uint64_t key = s_topk[r * MT_TOPK_MAX + j];
            tk.label[pt * tk.k + j] = (int64_t)(~(uint32_t)(key >> 16));
            if (tk.scores) tk.scores[pt * tk.k + j] = __ushort_as_half((unsigned short)(key & 0xffffu));
          }
          if ((lane & 3) == 0 && p.smax) p.smax[pt] = best[h];
        }
      }
    } else {
      // the four lanes of a row hold interleaved column pairs: the maximum with the smallest column wins
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int o = 1; o < 4; o <<= 1) {
          const float ob = __shfl_xor_sync(0xffffffffu, best[h], o);
          const int ok = __shfl_xor_sync(0xffffffffu, best_k[h], o);
          if (ob > best[h] || (ob == best[h] && ok < best_k[h])) { best[h] = ob; best_k[h] = ok; }
        }
        const int64_t pt = row0 + r_lo + 8 * h;
        if ((lane & 3) == 0 && pt < p.n_pts) {
          if (p.label) p.label[pt] = best_k[h];
          if (p.smax) p.smax[pt] = best[h];
        }
      }
    }
  }
  if constexpr (CE) {
    __syncthreads();
    if (warp == 0) {   // the block's partial in a fixed order: rows 4 lane .. 4 lane + 3, then a butterfly over the lanes
      double s = 0.0, c = 0.0;
#pragma unroll
      for (int j = 0; j < MT_M / 32; ++j) {
        const int r = (MT_M / 32) * lane + j;
        if (s_lab[r]) { s += (double)s_term[r]; c += 1.0; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        c += __shfl_xor_sync(0xffffffffu, c, o);
      }
      if (lane == 0) { ce.part[2 * blockIdx.x] = s; ce.part[2 * blockIdx.x + 1] = c; }
    }
    for (int b = tid; b < 3 * ce.classes; b += MT_THREADS)
      if (s_hist[b]) atomicAdd(&ce.areas[b], (unsigned long long)s_hist[b]);
  }
}

// one warp: the scene loss fp16(sum / rows) from the per-block partials, merged in block order (0 / 0 = NaN when no row
// is labelled)
__global__ void __launch_bounds__(32) k_match_ce_loss(const double *__restrict__ part, int64_t nblk, __half *loss) {
  const int lane = threadIdx.x;
  double s = 0.0, c = 0.0;
  for (int64_t b = lane; b < nblk; b += 32) { s += part[2 * b]; c += part[2 * b + 1]; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  if (lane == 0) *loss = __double2half(s / c);
}

template <int NP>
__global__ void __launch_bounds__(MT_THREADS, 1)
k_match_tc(const __grid_constant__ CUtensorMap tmT, const MatchTcParams p) {
  match_tc_body<NP, MT_PLAIN>(tmT, p, MatchTcVote{}, MatchTcCe{}, MatchTcTopk{});
}

template <int NP>
__global__ void __launch_bounds__(MT_THREADS, 1)
k_match_tc_vote(const __grid_constant__ CUtensorMap tmT, const MatchTcParams p, const MatchTcVote vo) {
  match_tc_body<NP, MT_VOTE>(tmT, p, vo, MatchTcCe{}, MatchTcTopk{});
}

template <int NP>
__global__ void __launch_bounds__(MT_THREADS, 1)
k_match_tc_ce(const __grid_constant__ CUtensorMap tmT, const MatchTcParams p, const MatchTcCe ce) {
  match_tc_body<NP, MT_CE>(tmT, p, MatchTcVote{}, ce, MatchTcTopk{});
}

template <int NP, bool F8 = false>
__global__ void __launch_bounds__(MT_THREADS, 1)
k_match_tc_topk(const __grid_constant__ CUtensorMap tmT, const MatchTcParams p, const MatchTcTopk tk) {
  match_tc_body<NP, MT_TOPK, F8>(tmT, p, MatchTcVote{}, MatchTcCe{}, tk);
}

static int launch_match_tc(const MatchTcParams &p, const MatchTcVote *vote, const MatchTcCe *ce, const MatchTcTopk *tk,
                           const void *text_f16, cudaStream_t stream) {
  CUtensorMap tmT;
  if (make_tmap_2b(&tmT, text_f16, (uint64_t)p.C, (uint64_t)p.k_text, MT_NW, 1)) return 1;
  const int NP = p.C / 64;
  const size_t smem = (size_t)NP * MT_M * 128 + MT_BSTAGES * MT_NW * 128 + 128 + 1024;
  const unsigned grid = (unsigned)ceil_div(p.n_pts, MT_M);
  if (tk != nullptr) {
    const size_t smem_tk = smem + (size_t)MT_M * MT_TOPK_MAX * 8;   // + the lists
    if (tk->row_exp && NP == 12) {
      OSB_SMEM_ATTR_ONCE((k_match_tc_topk<12, true>), 227 * 1024);
      k_match_tc_topk<12, true><<<grid, MT_THREADS, smem_tk, stream>>>(tmT, p, *tk);
    } else if (tk->row_exp) {
      OSB_SMEM_ATTR_ONCE((k_match_tc_topk<8, true>), 227 * 1024);
      k_match_tc_topk<8, true><<<grid, MT_THREADS, smem_tk, stream>>>(tmT, p, *tk);
    } else if (NP == 12) {
      OSB_SMEM_ATTR_ONCE(k_match_tc_topk<12>, 227 * 1024);
      k_match_tc_topk<12><<<grid, MT_THREADS, smem_tk, stream>>>(tmT, p, *tk);
    } else {
      OSB_SMEM_ATTR_ONCE(k_match_tc_topk<8>, 227 * 1024);
      k_match_tc_topk<8><<<grid, MT_THREADS, smem_tk, stream>>>(tmT, p, *tk);
    }
  } else if (ce != nullptr) {
    const size_t smem_ce = smem + 2 * MT_M * 4 + (size_t)3 * ce->classes * 4;   // + terms, flags, histogram
    if (NP == 12) {
      OSB_SMEM_ATTR_ONCE(k_match_tc_ce<12>, 227 * 1024);
      k_match_tc_ce<12><<<grid, MT_THREADS, smem_ce, stream>>>(tmT, p, *ce);
    } else {
      OSB_SMEM_ATTR_ONCE(k_match_tc_ce<8>, 227 * 1024);
      k_match_tc_ce<8><<<grid, MT_THREADS, smem_ce, stream>>>(tmT, p, *ce);
    }
    OSB_LAUNCH_CHECK();
    k_match_ce_loss<<<1, 32, 0, stream>>>(ce->part, grid, (__half *)ce->loss);
  } else if (vote != nullptr) {
    if (NP == 12) {
      OSB_SMEM_ATTR_ONCE(k_match_tc_vote<12>, 227 * 1024);
      k_match_tc_vote<12><<<grid, MT_THREADS, smem, stream>>>(tmT, p, *vote);
    } else {
      OSB_SMEM_ATTR_ONCE(k_match_tc_vote<8>, 227 * 1024);
      k_match_tc_vote<8><<<grid, MT_THREADS, smem, stream>>>(tmT, p, *vote);
    }
  } else if (NP == 12) {
    OSB_SMEM_ATTR_ONCE(k_match_tc<12>, 227 * 1024);
    k_match_tc<12><<<grid, MT_THREADS, smem, stream>>>(tmT, p);
  } else {
    OSB_SMEM_ATTR_ONCE(k_match_tc<8>, 227 * 1024);
    k_match_tc<8><<<grid, MT_THREADS, smem, stream>>>(tmT, p);
  }
  OSB_LAUNCH_CHECK();
  return 0;
}

static MatchTcParams match_tc_params(const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a,
                                     const float *sel_b, int c, const int64_t *inds_reverse, int64_t n_pts, int k_text,
                                     int normalize, void *scores_f16, int64_t *label, float *smax, void *feat_out_f16) {
  MatchTcParams p{};
  p.feat = feat; p.feat2 = (const __half *)feat2_f16; p.sel_a = sel_a; p.sel_b = sel_b;
  p.inds_reverse = inds_reverse; p.n_pts = n_pts; p.C = c; p.k_text = k_text;
  p.n_pass = (k_text + MT_NW - 1) / MT_NW;
  p.feat_is_f16 = feat_is_f16; p.normalize = normalize;
  p.scores = (__half *)scores_f16; p.label = label; p.smax = smax; p.feat_out = (__half *)feat_out_f16;
  return p;
}

// the [n_pts, K] epilogues: at most five passes
static int fill_match_tc(MatchTcParams &p, const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a,
                         const float *sel_b, int c, const int64_t *inds_reverse, int64_t n_pts, int k_text, int normalize,
                         void *scores_f16, int64_t *label, float *smax, void *feat_out_f16) {
  p = match_tc_params(feat, feat_is_f16, feat2_f16, sel_a, sel_b, c, inds_reverse, n_pts, k_text, normalize, scores_f16,
                      label, smax, feat_out_f16);
  OSB_CHECK(p.n_pass * MT_NW <= 512, "match: K_text=%d too large (at most 512 text rows)", k_text);
  return 0;
}

int match_tc_run(const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a, const float *sel_b, int c,
                 const int64_t *inds_reverse, int64_t n_pts, const void *text_f16, int k_text, int normalize,
                 void *scores_f16, int64_t *label, float *smax, void *feat_out_f16, cudaStream_t stream) {
  MatchTcParams p;
  if (fill_match_tc(p, feat, feat_is_f16, feat2_f16, sel_a, sel_b, c, inds_reverse, n_pts, k_text, normalize, scores_f16,
                    label, smax, feat_out_f16))
    return 1;
  return launch_match_tc(p, nullptr, nullptr, nullptr, text_f16, stream);
}

int match_tc_vote_run(const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a, const float *sel_b, int c,
                      const int64_t *inds_reverse, int64_t n_pts, const void *text_f16, int k_text, int normalize,
                      void *scores_f16, void *store_f16, int64_t *label_cur, int64_t *label_acc, cudaStream_t stream) {
  MatchTcParams p;
  if (fill_match_tc(p, feat, feat_is_f16, feat2_f16, sel_a, sel_b, c, inds_reverse, n_pts, k_text, normalize, scores_f16,
                    nullptr, nullptr, nullptr))
    return 1;
  const MatchTcVote vote{(__half *)store_f16, label_cur, label_acc,
                         (k_text % 2 == 0 && reinterpret_cast<uintptr_t>(store_f16) % 4 == 0) ? 1 : 0};
  return launch_match_tc(p, &vote, nullptr, nullptr, text_f16, stream);
}

int match_tc_ce_run(const void *feat, int feat_is_f16, int c, const int64_t *inds_reverse, int64_t n_pts, const void *text_f16,
                    int k_text, const void *label, int label_is_i64, int ignore, int classes, void *scores_f16, int64_t *pred,
                    void *loss_f16, uint64_t *areas, int32_t *bad, void *ws, cudaStream_t stream) {
  if (n_pts == 0) {   // no row: NaN loss, nothing counted
    k_match_ce_loss<<<1, 32, 0, stream>>>(nullptr, 0, (__half *)loss_f16);
    OSB_LAUNCH_CHECK();
    return 0;
  }
  MatchTcParams p;
  if (fill_match_tc(p, feat, feat_is_f16, nullptr, nullptr, nullptr, c, inds_reverse, n_pts, k_text, 0, scores_f16, pred,
                    nullptr, nullptr))
    return 1;
  const MatchTcCe ce{label, label_is_i64, ignore, classes, (double *)ws, (unsigned long long *)areas, bad, loss_f16};
  return launch_match_tc(p, nullptr, &ce, nullptr, text_f16, stream);
}

// streaming top-k: any number of passes (the caller bounds K); row_exp non-NULL: feat holds e4m3 codes (FP8 index rows)
int match_tc_topk_run(const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a, const float *sel_b, int c,
                      const int64_t *inds_reverse, int64_t n_pts, const void *text_f16, int k_text, int normalize, int topk,
                      void *scores_f16, int64_t *label, float *smax, void *feat_out_f16, const int8_t *row_exp,
                      cudaStream_t stream) {
  const MatchTcParams p = match_tc_params(feat, feat_is_f16, feat2_f16, sel_a, sel_b, c, inds_reverse, n_pts, k_text,
                                          normalize, nullptr, nullptr, smax, feat_out_f16);
  const MatchTcTopk tk{topk, (__half *)scores_f16, label, row_exp};
  return launch_match_tc(p, nullptr, nullptr, &tk, text_f16, stream);
}

}  // namespace osb
