// Open-vocabulary matching: voxel->point gather, optional L2 normalisation, fp16 product with the
// CLIP text embeddings, row max / argmax -- one pass over the features, nothing materialised at
// [N_pts, C].  Replaces the torch ops at run/evaluate.py:288-323.
//
// HBM-bound: 4*C bytes read per point (3 KB at C = 768) against 2*C*K flops; one warp owns one
// point, the text matrix (K*C*2 bytes, <= 737 KB at K = 480) stays in L1/L2.
//
// Label rule of every non-vote kernel (k_match_scores, k_match_ensemble, k_match_tc, k_folded_head_finish): the lowest
// column holding the largest non-NaN score, and 0 when no score is above -inf (a row of NaN and -inf only); smax is that
// largest non-NaN score, -inf when there is none.  Labels always lie in [0, K).  torch's CUDA `max(1)[1]`, which the
// reference takes, returns a NaN's index instead; the repeat vote and the validation cross-entropy (k_match_tc_ce) follow
// torch's CPU rule (vote.cuh).  So does the streaming top-k (k_match_tc_topk): NaN first, and its label 0 is vote.cuh's
// argmax; its smax is the rule above.
#include "common.cuh"
#include <algorithm>
#include <stdlib.h>

namespace osb {

template <int NP>  // half2 pairs per lane: C = 64 * NP
struct RowRegs {
  float v[2 * NP];
};

// load a feature row into registers as the fp16-rounded values the reference multiplies
template <int NP, bool F16, bool NORMALIZE>
__device__ __forceinline__ void load_row(const void *__restrict__ feat, int64_t row, int lane, RowRegs<NP> &r) {
  constexpr int C = 64 * NP;
  float ss = 0.f;
  if (F16) {
    const __half2 *p = reinterpret_cast<const __half2 *>(feat) + row * (C / 2);
#pragma unroll
    for (int j = 0; j < NP; ++j) {
      const float2 f = __half22float2(__ldg(p + lane + 32 * j));
      r.v[2 * j] = f.x; r.v[2 * j + 1] = f.y;
      ss += f.x * f.x + f.y * f.y;
    }
  } else {
    const float2 *p = reinterpret_cast<const float2 *>(feat) + row * (C / 2);
#pragma unroll
    for (int j = 0; j < NP; ++j) {
      const float2 f = __ldg(p + lane + 32 * j);
      r.v[2 * j] = f.x; r.v[2 * j + 1] = f.y;
      ss += f.x * f.x + f.y * f.y;
    }
  }
  if (NORMALIZE) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    float nrm = sqrtf(ss);
    if (F16) {
      // the reference takes norm / +1e-5 / division on an fp16 tensor (evaluate.py:303-305)
      nrm = __half2float(__float2half_rn(nrm));
      const float d = __half2float(__float2half_rn(nrm + 1e-5f));
#pragma unroll
      for (int j = 0; j < 2 * NP; ++j) r.v[j] = __half2float(__float2half_rn(r.v[j] / d));
    } else {
      const float d = nrm + 1e-5f;
#pragma unroll
      for (int j = 0; j < 2 * NP; ++j) r.v[j] = __half2float(__float2half_rn(r.v[j] / d));
    }
  } else if (!F16) {
#pragma unroll
    for (int j = 0; j < 2 * NP; ++j) r.v[j] = __half2float(__float2half_rn(r.v[j]));   // .half()
  }
}

template <int NP>
__device__ __forceinline__ void score_row(const RowRegs<NP> &r, const __half2 *__restrict__ text, int k_text, int lane,
                                          __half *__restrict__ scores_row, float &best, int &best_k) {
  constexpr int C = 64 * NP;
  best = -INFINITY;
  best_k = 0;
  for (int k = 0; k < k_text; ++k) {
    const __half2 *t = text + (int64_t)k * (C / 2);
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < NP; ++j) {
      const float2 f = __half22float2(__ldg(t + lane + 32 * j));
      acc = fmaf(r.v[2 * j], f.x, acc);
      acc = fmaf(r.v[2 * j + 1], f.y, acc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    const __half h = __float2half_rn(acc);
    const float s = __half2float(h);
    if (scores_row != nullptr && lane == 0) scores_row[k] = h;
    if (s > best) { best = s; best_k = k; }
  }
}

template <int NP, bool F16, bool NORMALIZE>
__global__ void __launch_bounds__(256)
k_match_scores(const void *__restrict__ feat, const int64_t *__restrict__ inds_reverse, int64_t n_pts,
               const __half2 *__restrict__ text, int k_text, __half *__restrict__ scores, int64_t *__restrict__ label,
               float *__restrict__ smax) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t p = warp; p < n_pts; p += nwarps) {
    const int64_t v = inds_reverse ? inds_reverse[p] : p;
    RowRegs<NP> r;
    load_row<NP, F16, NORMALIZE>(feat, v, lane, r);
    float best; int best_k;
    score_row<NP>(r, text, k_text, lane, scores ? scores + p * k_text : nullptr, best, best_k);
    if (lane == 0) {
      if (label) label[p] = best_k;
      if (smax) smax[p] = best;
    }
  }
}

template <int NP>
__global__ void __launch_bounds__(256)
k_match_ensemble(const float *__restrict__ feat3d, const __half *__restrict__ feat2d, const int64_t *__restrict__ inds_reverse,
                 int64_t n_pts, const float *__restrict__ smax3d, const float *__restrict__ smax2d,
                 const __half2 *__restrict__ text, int k_text, __half *__restrict__ scores, int64_t *__restrict__ label,
                 __half *__restrict__ feat_out) {
  constexpr int C = 64 * NP;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t p = warp; p < n_pts; p += nwarps) {
    const int64_t v = inds_reverse ? inds_reverse[p] : p;
    const bool use2d = smax3d[p] < smax2d[p];
    RowRegs<NP> r;
    if (use2d) load_row<NP, true, false>(feat2d, v, lane, r);
    else       load_row<NP, false, false>(feat3d, v, lane, r);
    if (feat_out) {
      __half2 *o = reinterpret_cast<__half2 *>(feat_out) + p * (C / 2);
#pragma unroll
      for (int j = 0; j < NP; ++j) o[lane + 32 * j] = __floats2half2_rn(r.v[2 * j], r.v[2 * j + 1]);
    }
    float best; int best_k;
    score_row<NP>(r, text, k_text, lane, scores ? scores + p * k_text : nullptr, best, best_k);
    if (lane == 0 && label) label[p] = best_k;
  }
}

// tensor-core implementation (match_tc.cu)
int match_tc_run(const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a, const float *sel_b, int c,
                 const int64_t *inds_reverse, int64_t n_pts, const void *text_f16, int k_text, int normalize,
                 void *scores_f16, int64_t *label, float *smax, void *feat_out_f16, cudaStream_t stream);

int match_tc_vote_run(const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a, const float *sel_b, int c,
                      const int64_t *inds_reverse, int64_t n_pts, const void *text_f16, int k_text, int normalize,
                      void *scores_f16, void *store_f16, int64_t *label_cur, int64_t *label_acc, cudaStream_t stream);
int match_tc_ce_run(const void *feat, int feat_is_f16, int c, const int64_t *inds_reverse, int64_t n_pts, const void *text_f16,
                    int k_text, const void *label, int label_is_i64, int ignore, int classes, void *scores_f16, int64_t *pred,
                    void *loss_f16, uint64_t *areas, int32_t *bad, void *ws, cudaStream_t stream);
int match_tc_topk_run(const void *feat, int feat_is_f16, const void *feat2_f16, const float *sel_a, const float *sel_b, int c,
                      const int64_t *inds_reverse, int64_t n_pts, const void *text_f16, int k_text, int normalize, int topk,
                      void *scores_f16, int64_t *label, float *smax, void *feat_out_f16, const int8_t *row_exp,
                      cudaStream_t stream);
// CUDA-core repeat vote (vote.cu)
int vote_accumulate_run(const void *src, int src_is_f16, const int64_t *inds_reverse, int64_t n_pts, int k, void *store,
                        int64_t *label_cur, int64_t *label_acc, cudaStream_t stream);

static bool use_simt() {   // OSB_MATCH_SIMT=1 selects the CUDA-core kernels below (cross-check path)
  static int v = -1;
  if (v < 0) { const char *e = getenv("OSB_MATCH_SIMT"); v = (e && e[0] == '1') ? 1 : 0; }
  return v == 1;
}

static unsigned match_grid(int64_t n_pts) {
  return (unsigned)std::min<int64_t>(ceil_div(n_pts, 8), 132 * 8);
}

}  // namespace osb

using namespace osb;

extern "C" {

int osb_match_scores(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse,
                     int64_t n_pts, const void *text_f16, int32_t k_text, int32_t normalize, void *scores_f16,
                     int64_t *label, float *smax, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(c == 512 || c == 768, "osb_match_scores: feature width %d unsupported (OpenScene uses 512 / 768)", c);
  OSB_CHECK(k_text >= 1 && k_text <= 480, "osb_match_scores: K_text=%d outside 1..480", k_text);
  OSB_CHECK(n_vox > 0, "osb_match_scores: bad shape");
  if (n_pts == 0) return 0;
  if (!use_simt())
    return match_tc_run(feat, feat_is_f16, nullptr, nullptr, nullptr, c, inds_reverse, n_pts, text_f16, k_text, normalize,
                        scores_f16, label, smax, nullptr, stream);
  const unsigned grid = match_grid(n_pts);
  const __half2 *text = (const __half2 *)text_f16;
  __half *scores = (__half *)scores_f16;
#define OSB_MS(NP, F16, NRM) \
  k_match_scores<NP, F16, NRM><<<grid, 256, 0, stream>>>(feat, inds_reverse, n_pts, text, k_text, scores, label, smax)
  if (c == 768) {
    if (feat_is_f16) { if (normalize) OSB_MS(12, true, true); else OSB_MS(12, true, false); }
    else             { if (normalize) OSB_MS(12, false, true); else OSB_MS(12, false, false); }
  } else {
    if (feat_is_f16) { if (normalize) OSB_MS(8, true, true); else OSB_MS(8, true, false); }
    else             { if (normalize) OSB_MS(8, false, true); else OSB_MS(8, false, false); }
  }
#undef OSB_MS
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_match_ensemble(const float *feat3d, const void *feat2d_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse,
                       int64_t n_pts, const float *smax3d, const float *smax2d, const void *text_f16, int32_t k_text,
                       void *scores_f16, int64_t *label, void *feat_out_f16, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(c == 512 || c == 768, "osb_match_ensemble: feature width %d unsupported", c);
  OSB_CHECK(k_text >= 1 && k_text <= 480, "osb_match_ensemble: K_text=%d outside 1..480", k_text);
  OSB_CHECK(n_vox > 0, "osb_match_ensemble: bad shape");
  if (n_pts == 0) return 0;
  if (!use_simt())
    return match_tc_run(feat3d, 0, feat2d_f16, smax3d, smax2d, c, inds_reverse, n_pts, text_f16, k_text, 0, scores_f16, label,
                        nullptr, feat_out_f16, stream);
  const unsigned grid = match_grid(n_pts);
  if (c == 768)
    k_match_ensemble<12><<<grid, 256, 0, stream>>>(feat3d, (const __half *)feat2d_f16, inds_reverse, n_pts, smax3d, smax2d,
                                                   (const __half2 *)text_f16, k_text, (__half *)scores_f16, label,
                                                   (__half *)feat_out_f16);
  else
    k_match_ensemble<8><<<grid, 256, 0, stream>>>(feat3d, (const __half *)feat2d_f16, inds_reverse, n_pts, smax3d, smax2d,
                                                  (const __half2 *)text_f16, k_text, (__half *)scores_f16, label,
                                                  (__half *)feat_out_f16);
  OSB_LAUNCH_CHECK();
  return 0;
}

// Repeat vote.  The tensor-core path adds the fp16 scores into the store in the epilogue of the product (the scores reach
// HBM only when asked for); OSB_MATCH_SIMT=1 writes them to a scratch buffer with the CUDA-core kernels above and votes
// with k_vote_accumulate.  Both give the same bits.
static int match_vote_simt(int rc, void *scratch, bool own, int64_t n_pts, int32_t k_text, void *store_f16,
                           int64_t *label_cur, int64_t *label_acc, cudaStream_t stream) {
  if (rc == 0) rc = vote_accumulate_run(scratch, 1, nullptr, n_pts, k_text, store_f16, label_cur, label_acc, stream);
  if (own) cudaFreeAsync(scratch, stream);
  return rc;
}

static int check_vote_args(const char *fn, int32_t c, int32_t k_text, int64_t n_vox, int64_t n_pts, const void *store_f16) {
  OSB_CHECK(c == 512 || c == 768, "%s: feature width %d unsupported (OpenScene uses 512 / 768)", fn, c);
  OSB_CHECK(k_text >= 1 && k_text <= 480, "%s: K_text=%d outside 1..480", fn, k_text);
  OSB_CHECK(n_vox > 0 && n_pts >= 0, "%s: bad shape", fn);
  OSB_CHECK(store_f16 != nullptr, "%s: null store", fn);
  return 0;
}

int osb_match_vote(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse,
                   int64_t n_pts, const void *text_f16, int32_t k_text, int32_t normalize, void *scores_f16,
                   void *store_f16, int64_t *label_cur, int64_t *label_acc, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (check_vote_args("osb_match_vote", c, k_text, n_vox, n_pts, store_f16)) return 1;
  if (n_pts == 0) return 0;
  if (!use_simt())
    return match_tc_vote_run(feat, feat_is_f16, nullptr, nullptr, nullptr, c, inds_reverse, n_pts, text_f16, k_text,
                             normalize, scores_f16, store_f16, label_cur, label_acc, stream);
  void *scratch = scores_f16;
  if (scratch == nullptr) OSB_CUDA(cudaMallocAsync(&scratch, (size_t)n_pts * k_text * sizeof(__half), stream));
  const int rc = osb_match_scores(feat, feat_is_f16, n_vox, c, inds_reverse, n_pts, text_f16, k_text, normalize, scratch,
                                  nullptr, nullptr, stream_);
  return match_vote_simt(rc, scratch, scores_f16 == nullptr, n_pts, k_text, store_f16, label_cur, label_acc, stream);
}

int osb_match_ensemble_vote(const float *feat3d, const void *feat2d_f16, int64_t n_vox, int32_t c,
                            const int64_t *inds_reverse, int64_t n_pts, const float *smax3d, const float *smax2d,
                            const void *text_f16, int32_t k_text, void *scores_f16, void *store_f16, int64_t *label_cur,
                            int64_t *label_acc, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  if (check_vote_args("osb_match_ensemble_vote", c, k_text, n_vox, n_pts, store_f16)) return 1;
  if (n_pts == 0) return 0;
  if (!use_simt())
    return match_tc_vote_run(feat3d, 0, feat2d_f16, smax3d, smax2d, c, inds_reverse, n_pts, text_f16, k_text, 0,
                             scores_f16, store_f16, label_cur, label_acc, stream);
  void *scratch = scores_f16;
  if (scratch == nullptr) OSB_CUDA(cudaMallocAsync(&scratch, (size_t)n_pts * k_text * sizeof(__half), stream));
  const int rc = osb_match_ensemble(feat3d, feat2d_f16, n_vox, c, inds_reverse, n_pts, smax3d, smax2d, text_f16, k_text,
                                    scratch, nullptr, nullptr, stream_);
  return match_vote_simt(rc, scratch, scores_f16 == nullptr, n_pts, k_text, store_f16, label_cur, label_acc, stream);
}

// Validation tail of run/distill.py (:419-431) in the epilogue of the tensor-core product; no CUDA-core route.
int osb_match_ce(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse, int64_t n_pts,
                 const void *text_f16, int32_t k_text, const void *label, int32_t label_is_i64, int32_t ignore_index,
                 int32_t classes, void *scores_f16, int64_t *pred, void *loss_f16, uint64_t *areas, int32_t *bad_labels,
                 void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(c == 512 || c == 768, "osb_match_ce: feature width %d unsupported (OpenScene uses 512 / 768)", c);
  OSB_CHECK(k_text >= 1 && k_text <= 480, "osb_match_ce: K_text=%d outside 1..480", k_text);
  OSB_CHECK(classes >= 1 && classes <= 512, "osb_match_ce: classes=%d outside 1..512", classes);
  OSB_CHECK(n_vox > 0 && n_pts >= 0, "osb_match_ce: bad shape (n_vox=%lld, n_pts=%lld)", (long long)n_vox, (long long)n_pts);
  OSB_CHECK(label_is_i64 == 0 || label_is_i64 == 1, "osb_match_ce: label_is_i64 must be 0 or 1");
  OSB_CHECK(feat && text_f16 && (label || n_pts == 0) && loss_f16 && areas && bad_labels,
            "osb_match_ce: null features, text, labels, loss, areas or bad-label flag");
  const size_t need = (size_t)16 * ceil_div(n_pts, 128);
  OSB_CHECK(need == 0 || (ws != nullptr && ws_bytes >= need && ((uintptr_t)ws & 7) == 0),
            "osb_match_ce: 8-byte aligned workspace of %zu bytes required (got %zu)", need, ws_bytes);
  return match_tc_ce_run(feat, feat_is_f16, c, inds_reverse, n_pts, text_f16, k_text, label, label_is_i64, ignore_index,
                         classes, scores_f16, pred, loss_f16, areas, bad_labels, ws, stream);
}

// Streaming top-k over any number of 96-row passes; tensor-core route only.
static int check_topk_args(const char *fn, int32_t c, int32_t k_text, int32_t topk, int64_t n_vox, int64_t n_pts,
                           const void *text_f16, const int64_t *label) {
  OSB_CHECK(c == 512 || c == 768, "%s: feature width %d unsupported (OpenScene uses 512 / 768)", fn, c);
  OSB_CHECK(k_text >= 1 && k_text <= OSB_MATCH_TOPK_MAX_TEXT, "%s: K_text=%d outside 1..%d", fn, k_text,
            OSB_MATCH_TOPK_MAX_TEXT);
  OSB_CHECK(topk >= 1 && topk <= std::min(8, k_text), "%s: topk=%d outside 1..min(8, K_text=%d)", fn, topk, k_text);
  OSB_CHECK(n_vox > 0 && n_pts >= 0, "%s: bad shape (n_vox=%lld, n_pts=%lld)", fn, (long long)n_vox, (long long)n_pts);
  OSB_CHECK(text_f16 != nullptr, "%s: NULL text", fn);
  OSB_CHECK(label != nullptr, "%s: NULL label", fn);
  return 0;
}

int osb_match_topk(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse,
                   int64_t n_pts, const void *text_f16, int32_t k_text, int32_t normalize, int32_t topk, void *scores_f16,
                   int64_t *label, float *smax, void *stream_) {
  if (check_topk_args("osb_match_topk", c, k_text, topk, n_vox, n_pts, text_f16, label)) return 1;
  OSB_CHECK(feat != nullptr, "osb_match_topk: NULL features");
  if (n_pts == 0) return 0;
  return match_tc_topk_run(feat, feat_is_f16, nullptr, nullptr, nullptr, c, inds_reverse, n_pts, text_f16, k_text, normalize,
                           topk, scores_f16, label, smax, nullptr, nullptr, (cudaStream_t)stream_);
}

// osb_match_topk over FP8 scene-index rows d = code * 2^e (no point expansion, no normalisation)
int osb_match_topk_f8(const void *codes_f8, const int8_t *row_exp, int64_t n_rows, int32_t c, const void *text_f16,
                      int32_t k_text, int32_t topk, void *scores_f16, int64_t *label, float *smax, void *stream_) {
  if (check_topk_args("osb_match_topk_f8", c, k_text, topk, n_rows, n_rows, text_f16, label)) return 1;
  OSB_CHECK(codes_f8 != nullptr && row_exp != nullptr, "osb_match_topk_f8: NULL codes or row exponents");
  OSB_CHECK(n_rows < (int64_t(1) << 31), "osb_match_topk_f8: N=%lld outside 1..2^31-1", (long long)n_rows);
  OSB_CHECK(((uintptr_t)codes_f8 & 15) == 0 && ((uintptr_t)text_f16 & 15) == 0,
            "osb_match_topk_f8: codes and text must be 16-byte aligned");
  return match_tc_topk_run(codes_f8, 1, nullptr, nullptr, nullptr, c, nullptr, n_rows, text_f16, k_text, 0, topk,
                           scores_f16, label, smax, nullptr, row_exp, (cudaStream_t)stream_);
}

int osb_match_ensemble_topk(const float *feat3d, const void *feat2d_f16, int64_t n_vox, int32_t c,
                            const int64_t *inds_reverse, int64_t n_pts, const float *sel_a, const float *sel_b,
                            const void *text_f16, int32_t k_text, int32_t topk, void *scores_f16, int64_t *label,
                            void *feat_out_f16, void *stream_) {
  if (check_topk_args("osb_match_ensemble_topk", c, k_text, topk, n_vox, n_pts, text_f16, label)) return 1;
  OSB_CHECK(feat3d && feat2d_f16 && sel_a && sel_b, "osb_match_ensemble_topk: NULL features or row maxima");
  if (n_pts == 0) return 0;
  return match_tc_topk_run(feat3d, 0, feat2d_f16, sel_a, sel_b, c, inds_reverse, n_pts, text_f16, k_text, 0, topk, scores_f16,
                           label, nullptr, feat_out_f16, nullptr, (cudaStream_t)stream_);
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// Folded head (optional fast path, openscene_b200/engine.py: forward_scores): the final 1x1x1 convolution
// f = x W (96 -> 768) and the cosine product with the text matrix T are re-associated,
//     f . t_k = x . (W t_k) = x . U_k,      |f|^2 = x (W W^T) x^T = |x L|^2   (W W^T = L L^T, Cholesky),
// so one 96 -> (96 + K) convolution produces z = [x L | x U] and this kernel finishes a row:
//     score_k = fp16( (x.U_k) / (|x L| + 1e-5) ),  label = argmax_k.
namespace osb {
__global__ void k_folded_head_finish(const float *__restrict__ z, int64_t n, int ld, int c_norm, int k_text,
                                     __half *__restrict__ scores, int64_t *__restrict__ label, float *__restrict__ smax) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t p = warp; p < n; p += nwarps) {
    const float *row = z + p * ld;
    float ss = 0.f;
    for (int c = lane; c < c_norm; c += 32) { const float v = __ldg(row + c); ss = fmaf(v, v, ss); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
    const float d = sqrtf(ss) + 1e-5f;
    float best = -INFINITY;
    int best_k = 0;          // the label rule above: 0 when no score is above -inf
    for (int k = lane; k < k_text; k += 32) {
      const __half h = __float2half_rn(__ldg(row + c_norm + k) / d);
      if (scores) scores[p * k_text + k] = h;
      const float s = __half2float(h);
      if (s > best) { best = s; best_k = k; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int ok = __shfl_xor_sync(0xffffffffu, best_k, o);
      if (ob > best || (ob == best && ok < best_k)) { best = ob; best_k = ok; }
    }
    if (lane == 0) {
      if (label) label[p] = best_k;
      if (smax) smax[p] = best;
    }
  }
}
}  // namespace osb

extern "C" int osb_folded_head_finish(const float *z, int64_t n, int32_t ld, int32_t c_norm, int32_t k_text, void *scores_f16,
                                      int64_t *label, float *smax, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n > 0 && c_norm > 0 && k_text > 0 && ld >= c_norm + k_text, "osb_folded_head_finish: bad shape");
  const unsigned grid = (unsigned)std::min<int64_t>(osb::ceil_div(n, 8), 132 * 8);
  osb::k_folded_head_finish<<<grid, 256, 0, stream>>>(z, n, ld, c_norm, k_text, (__half *)scores_f16, label, smax);
  OSB_LAUNCH_CHECK();
  return 0;
}
