/*
 * osb200.h -- C ABI of libosb200.so, the H100 (sm_90a) sparse-3D-convolution + open-vocabulary
 * matching engine that replaces the MinkowskiEngine native backend and the driver-side torch ops on
 * OpenScene's hot path.
 *
 * What each group replaces in the reference (paths relative to the reference root):
 *   osb_coordset_* / osb_kernel_map_*   the coordinate manager inside MinkowskiEngine that
 *        `ME.SparseTensor(feat, coords)` (run/evaluate.py:284, run/distill.py:316) and every
 *        `ME.MinkowskiConvolution(..., kernel_size=k, stride=s)` (models/mink_unet.py:47-113) drive:
 *        coordinate hash, tensor-stride sets, per-offset kernel maps.
 *   osb_conv_*                          `MinkowskiConvolution.forward` / `MinkowskiConvolutionTranspose.forward`
 *        (gather -> GEMM -> scatter-add per sparse-conv layer; models/mink_unet.py:116-174) and their autograd
 *        backward (run/distill.py:333).
 *        `MinkowskiBatchNorm` (eval) / `MinkowskiReLU` / the BasicBlock residual / `ME.cat` have no entry points of their
 *        own: they are arguments of osb_conv_* (scale/shift, relu, res, src1), folded into the convolution's epilogue
 *        (models/mink_unet.py:50,114,147).
 *   osb_match_*                         `predictions[inds_reverse]`, `x/(|x|+1e-5)`, `.half() @ text_features.t()`,
 *        `torch.max(pred,1)` (run/evaluate.py:288-323); osb_match_ce also the cross-entropy loss and
 *        `intersectionAndUnionGPU` of run/distill.py: validate() (:419-431) in the same pass.
 *   osb_voxelize_*                      `Voxelizer.voxelize` + `sparse_quantize`/`fnv_hash_vec`
 *        (dataset/voxelizer.py:97-140, dataset/voxelization_utils.py:9-22,44-137).
 *   osb_fusion_*                        the multi-view fusion loop: `PointCloudToImageMapper.compute_mapping`
 *        (scripts/feature_fusion/fusion_util.py:102-139) + the running mean of
 *        scripts/feature_fusion/scannet_openseg.py:74-108 (SURVEY.md 8f rank 2).
 *   osb_feature_remap                   the fused-feature index remap of `FusedFeatureLoader.__getitem__`
 *        (dataset/feature_loader.py:101-172) (SURVEY.md 8f rank 3).
 *   osb_confusion_* / osb_intersection_union   `confusion_matrix` (util/metric.py:9-25) and
 *        `intersectionAndUnionGPU` (util/util.py:132-145) (SURVEY.md 8f rank 4).
 *
 * Conventions
 *   - every pointer is a raw DEVICE pointer unless the name ends in `_host`;
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises
 *     unless documented ("SYNC");
 *   - the CALLER allocates every output and workspace (sizes via the *_workspace_bytes queries), so
 *     memory stays in the caller's allocator; the library keeps no per-call state (the only process-wide state are the
 *     tuning knobs of osb_tuning_set, which never change results);
 *   - every function returns 0 on success, non-zero on failure; osb_last_error() returns a
 *     thread-local description; no exception crosses the ABI;
 *   - there is no CPU fallback: on a machine without an sm_90 GPU every compute entry point fails.
 */
#ifndef OSB200_H
#define OSB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OSB_VERSION 100

/* ------------------------------------------------------------------ misc */
int         osb_version(void);
const char *osb_last_error(void);
/* sm count, compute capability of the current device. */
int osb_device_info(int *sm_count, int *cc_major, int *cc_minor);
/* number of kernels this library has launched in this process (bench.py's `gpu_launches`). */
int64_t osb_launch_count(void);
/* SM clock in MHz measured on the device (clock64 against %globaltimer over ~20 us); *mhz_dev is a device float. */
int osb_measure_sm_mhz(float *mhz_dev, void *stream);

/* --------------------------------------------------------- coordinate sets
 * A coordinate is an int32 row (b, x, y, z).  Valid range: 0 <= b < 1024, |x|,|y|,|z| < 2^17 - 256.
 * Internally rows are kept in Morton order (b major) -- the "internal order"; `perm[r]` is the
 * caller's row of internal row r.
 *
 * Hash table: `cap` slots of 16 bytes {uint64 key, int32 row, int32 pad}, cap a power of two >= 2n.
 */
size_t osb_coordset_workspace_bytes(int64_t n);

/* Build the tensor-stride-1 set from caller-order coordinates.
 *   coords      in  int32 [n,4]
 *   coords_int  out int32 [n,4]   coordinates in internal (Morton) order
 *   perm        out int32 [n]     internal row -> caller row
 *   inv_perm    out int32 [n]     caller row  -> internal row
 *   slots       out 16B  [cap]    hash table over coords_int
 *   status_host out int32 [6]     HOST: [0] bit0 = coordinate out of range, bit1 = duplicate coordinate; [1] reserved;
 *                                 [2..5] = OR (lo, hi word) and AND (lo, hi word) of the 64-bit Morton keys
 *                                 b<<54 | interleave(x+2^17, y+2^17, z+2^17) -- sizes the occupancy grid below
 *   slots may be NULL (no hash table wanted: the caller uses an occupancy grid)
 * SYNC: waits for `stream` to deliver status_host. */
int osb_coordset_build(const int32_t *coords, int64_t n, int32_t *coords_int, int32_t *perm, int32_t *inv_perm,
                       void *slots, int64_t cap, int32_t *status_host, void *ws, size_t ws_bytes, void *stream);

/* Coarser set: unique(floor(c / new_ts) * new_ts) per batch index, Morton ordered.
 *   coords_fine   in  int32 [n,4] (internal order)
 *   new_ts        absolute tensor stride of the coarse set (any integer >= 1)
 *   coords_coarse out int32 [<=n,4]
 *   parent_of     out int32 [n]     fine row -> coarse row
 *   n_coarse_host out int64 [1]     HOST
 * SYNC. */
int osb_coordset_stride(const int32_t *coords_fine, int64_t n, int32_t new_ts, int32_t *coords_coarse,
                        int32_t *parent_of, int64_t *n_coarse_host, void *ws, size_t ws_bytes, void *stream);

/* The whole stride-2 pyramid of a U-Net encoder in one call (2 host syncs instead of 2 per level): tensor-stride-1 set
 * as osb_coordset_build, plus `n_levels` coarser sets with tensor strides 2, 4, ..., 2^n_levels.  Children are Morton
 * sorted, so parents of a power-of-two stride are already in order: no sort, level counts stay on the device.
 *   coords_lvl  out int32 [n_levels][n,4]   coarse sets, upper-bound sized (use the first n_host[l+1] rows of slab l)
 *   parent_lvl  out int32 [n_levels][n]     parent_lvl[l][r]: row of level-l row r in level l+1
 *   n_host      out int64 [n_levels+1]      HOST: rows per level;  status_host as osb_coordset_build
 * SYNC. */
int osb_coordset_pyramid(const int32_t *coords, int64_t n, int32_t n_levels, int32_t *coords_int, int32_t *perm,
                         int32_t *inv_perm, void *slots, int64_t cap, int32_t *coords_lvl, int32_t *parent_lvl,
                         int64_t *n_host, int32_t *status_host, void *ws, size_t ws_bytes, void *stream);

/* (Re)build a hash table over internal-order coordinates. */
int osb_hash_build(const int32_t *coords_int, int64_t n, void *slots, int64_t cap, void *stream);

/* Kernel map in output-stationary form: nbr[k*n_out + o] = input row at c_out[o] + delta_k*step, or -1.
 * Offsets enumerate x fastest; odd kernel sizes are centred, even ones use delta in {0..ks-1}
 * (region convention of the generalised sparse convolution; SURVEY.md 8a a6).
 *   pairs_per_k   out int32 [K] (may be NULL): number of valid pairs per offset. */
int osb_kernel_map_build(const int32_t *coords_out, int64_t n_out, const void *slots_in, int64_t cap_in,
                         int32_t ks_x, int32_t ks_y, int32_t ks_z, int32_t step, int32_t *nbr,
                         int32_t *pairs_per_k, void *stream);

/* Swap the roles of input and output: nbr_t[k*n_in + i] = o  iff  nbr[k*n_out + o] = i  (else -1). */
int osb_kernel_map_transpose(const int32_t *nbr, int64_t n_out, int32_t K, int32_t *nbr_t, int64_t n_in,
                             void *stream);

/* ----------------------------------------------------------- sparse conv
 * Generic fp32 path (CUDA cores; any channel counts).  out[o,:] = sum_k in[nbr[k][o],:] @ W[k]
 *   in   fp32 [n_in, cin] (row stride ld_in floats)     w  fp32 [K, cin, cout]
 *   out  fp32 [n_out, cout]
 *   transpose_w != 0: use W[k]^T, i.e. w is [K, cout, cin] (dgrad).
 *   nbr NULL: the identity map (K == 1).  Refused before any launch: ld_in < cin, NULL in / w / out. */
int osb_conv_fwd_f32(const float *in, int64_t ld_in, const int32_t *nbr, int64_t n_out, int32_t K,
                     const float *w, int32_t cin, int32_t cout, int32_t transpose_w, float *out, void *stream);

/* Weight gradient: gw[k] = sum_o in[nbr[k][o],:]^T gout[o,:]   (gw fp32 [K,cin,cout], overwritten; in rows of cin floats).
 * nbr NULL: the identity map (K == 1).  Refused before any launch or memset: NULL in / gout / gw. */
int osb_conv_wgrad_f32(const float *in, const int32_t *nbr, int64_t n_out, int32_t K, const float *gout,
                       int32_t cin, int32_t cout, float *gw, void *stream);

/* Weight gradient on tensor cores (run/distill.py:333): gw[k] = sum_o x[nbr[k][o],:]^T gout[o,:] with both operands in the
 * split layout (x_split [n_in, cin], gout_split [n_out, cout]); gw fp32 [K,cin,cout] is overwritten.  Every product is the
 * full (hi+lo)(hi+lo) expansion on kind::f16 MMAs with fp32 accumulation; partial tiles are reduced in a fixed order
 * (bit-reproducible, no atomics).  ws: osb_conv_wgrad_tc_workspace_bytes(...) bytes. */
size_t osb_conv_wgrad_tc_workspace_bytes(int64_t n_out, int32_t K, int32_t cin, int32_t cout);
int osb_conv_wgrad_tc(const void *x_split, int32_t cin, int64_t n_in, const int32_t *nbr, int64_t n_out, int32_t K,
                      const void *gout_split, int32_t cout, float *gw, void *ws, size_t ws_bytes, void *stream);

/* Tensor-core path (wgmma, bf16x3 split-fp32 operands, fp32 accumulation in registers).
 *
 * Activation "split" layout: a row of C channels (C % 32 == 0) is 4*C bytes; every 32-channel block is
 * one 128-byte line [bf16 hi x32 | bf16 lo x32] with hi = bf16_rn(v), lo = bf16_rn(v - hi).
 * Packed weights (osb_conv_pack_weights): per offset k, cout_pad rows of the same split layout over
 * cin, i.e. the K-major B operand.
 *
 *   src0/src1   split rows, c0 and c1 channels (src1 may be NULL with c1 = 0): the conv input is the
 *               column concatenation [src0 | src1] -- `ME.cat` without materialising it
 *   nbr         int32 [K, n_out]  (NULL with K == 1 means identity: a 1x1x1 conv)
 *   wpack       packed weights for cin = c0 + c1
 *   scale/shift fp32 [cout] or NULL: y = acc*scale + shift   (eval-mode BatchNorm folded)
 *   res         residual added before ReLU: split rows [n_out, cout] or NULL
 *   relu        != 0 applies max(y, 0)
 *   out_split   split rows [n_out, cout] or NULL
 *   out_f32     fp32 [n_out, cout] or NULL; out_row_map (int32 [n_out] or NULL) scatters fp32 rows:
 *               row o is written to out_f32[out_row_map[o]]
 *   flags       bit0: launch with programmatic stream serialization (PDL).  The kernel's prologue (barrier
 *               set-up, loading `nbr`, scale, shift) then overlaps the tail of the previous kernel in `stream`; it
 *               waits for that kernel before touching src*, res, ws or any output.  Only legal when nbr / wpack /
 *               scale / shift were NOT produced by the immediately preceding kernel in the stream.
 */
size_t osb_conv_packed_weight_bytes(int32_t K, int32_t cin, int32_t cout);
/* Scratch osb_conv_fwd_tc needs for this shape: small problems are split over the (offset, channel-block)
 * sequence across CTAs (fp32 partials + a deterministic reduce kernel); 0 when no split is used. */
size_t osb_conv_tc_workspace_bytes(int64_t n_out, int32_t K, int32_t cin, int32_t cout);
int osb_conv_pack_weights(const float *w, int32_t K, int32_t cin, int32_t cout, int32_t transpose_w,
                          void *wpack, void *stream);
int osb_conv_fwd_tc(const void *src0, int32_t c0, int64_t n_src0, const void *src1, int32_t c1, int64_t n_src1,
                    const int32_t *nbr, int64_t n_out, int32_t K, const void *wpack, int32_t cout,
                    const float *scale, const float *shift, const void *res, int32_t relu, void *out_split,
                    float *out_f32, const int32_t *out_row_map, void *ws, size_t ws_bytes, int32_t flags, void *stream);

/* Transposed stride-2 convolution (`MinkowskiConvolutionTranspose(kernel_size=2, stride=2)`, models/mink_unet.py:79-101) as a
 * dense GEMM over the coarse rows followed by a scatter to the children: wpack = osb_conv_pack_weights of the
 * [1, cin, kvol*cout] matrix (column block k = W[k]); down_nbr = int32 [kvol, n_coarse], the kernel map of the matching
 * strided convolution (child row of parent o through offset k, -1 if absent).  out_* have one row per FINE voxel and
 * `cout` channels; every fine row is written exactly once.  scale/shift/relu/flags as osb_conv_fwd_tc. */
int osb_convtr_fwd_tc(const void *src, int32_t cin, int64_t n_coarse, const int32_t *down_nbr, int32_t kvol, const void *wpack,
                      int32_t cout, const float *scale, const float *shift, int32_t relu, void *out_split, float *out_f32,
                      int32_t flags, void *stream);


/* ----------------------------------------------------------- persistent convolution chains (conv_chain.cu)
 * Second-generation tensor-core path: ONE launch executes a list of convolution layers (`MinkowskiConvolution` /
 * `MinkowskiConvolutionTranspose` forwards of consecutive modules of models/mink_unet.py:116-174, BasicBlock included) with
 * one persistent CTA per SM, producer warps and two consumer warpgroups (wgmma + epilogue), split-K reduced inside the
 * kernel and grid barriers between dependent layers.  Same arithmetic and the same argument meaning as osb_conv_fwd_tc.
 *
 * A layer is described by an opaque record of osb_conv_desc_bytes() bytes, filled on the HOST by osb_conv_desc_fill; the
 * launch passes the records to the kernel as launch parameters (16 layers per launch, longer lists in several launches).
 *   wtiles          osb_conv_pack_weight_tiles(w [K,cin,cout]) -- tile-major, pre-swizzled B operands
 *   cmap/cmap_cout  non-NULL: dense transposed stride-2 convolution as in osb_convtr_fwd_tc (wtiles of the [1,cin,kvol*cout]
 *                   matrix, cout = kvol*cmap_cout, cmap = the stride-2 map [kvol, n_out] of the matching strided conv)
 *   ws / ws_bytes   scratch for split-K partials, osb_conv_chain_workspace_bytes(...) bytes (0 = not split).  Consecutive
 *                   split layers without a barrier between them need different scratch
 *   barrier_before  != 0: this layer reads (src*, res) what an earlier layer of the SAME launch wrote
 *   grid_barrier    2 x uint32 in device memory, zeroed once when allocated (never reset afterwards); required when any
 *                   layer of the launch is split or asks for a barrier.  One launch at a time may use it.
 *   flags           bit0: PDL, as in osb_conv_fwd_tc */
size_t osb_conv_desc_bytes(void);
size_t osb_conv_weight_tiles_bytes(int32_t K, int32_t cin, int32_t cout);
int osb_conv_pack_weight_tiles(const float *w, int32_t K, int32_t cin, int32_t cout, int32_t transpose_w, void *wtiles,
                               void *stream);
int osb_conv_chain_grid(void);
size_t osb_conv_chain_workspace_bytes(int64_t n_out, int32_t K, int32_t cin, int32_t cout);
int osb_conv_desc_fill(void *desc_host, const void *src0, int32_t c0, const void *src1, int32_t c1, const int32_t *nbr,
                       int64_t n_out, int32_t K, const void *wtiles, int32_t cout, const float *scale, const float *shift,
                       const void *res, int32_t relu, void *out_split, float *out_f32, const int32_t *out_row_map,
                       const int32_t *cmap, int32_t cmap_cout, void *ws, size_t ws_bytes, int32_t barrier_before);
int osb_conv_chain_launch(const void *descs_host, int32_t n_layers, void *grid_barrier, int32_t flags, void *stream);

/* Process-wide tuning knobs (tile shapes, ring depths, split factors, profiling hooks).  They select between
 * equivalent schedules and never change results; unknown names fail.  Names: see csrc/conv_chain.cu, csrc/conv_tc.cu. */
int osb_tuning_set(const char *name, int64_t value);

/* Stem: fused kernel-map probe + conv for tiny cin (<= 3) and cout <= 32, fp32 FMA.  One launch replaces the
 * 5x5x5 map build (125 probes / voxel) and the 3->32 convolution of `conv0p1s1`.
 *   in  fp32 [n, cin] internal order;  w fp32 [K, cin, cout];  epilogue as osb_conv_fwd_tc. */
int osb_conv_stem_fused(const float *in, int32_t cin, const int32_t *coords, int64_t n, const void *slots,
                        int64_t cap, int32_t ks, int32_t step, const float *w, int32_t cout, const float *scale,
                        const float *shift, int32_t relu, void *out_split, float *out_f32, void *stream);

/* Train-mode BatchNorm on split rows (`MinkowskiBatchNorm` / nn.BatchNorm1d with training=True over the [n, C] feature matrix;
 * run/distill.py's validate() runs the network this way under no_grad).  The convolution before it runs with scale/shift =
 * NULL and relu = 0; these two calls normalise its raw output.
 *
 * osb_bn_batch_stats: per-channel mean and biased variance over all n rows (every batch index together), then
 *   scale = weight / sqrt(var + eps), shift = bias - mean * scale               (fp32 [c] outputs)
 *   running_mean = (1 - m) running_mean + m mean, running_var = (1 - m) running_var + m var n / (n - 1),
 *   num_batches_tracked += 1                                                   (in place, fp32 [c] / int64 [1])
 * with m = momentum, or m = 1 / num_batches_tracked (after the increment) when momentum < 0 (momentum=None).  Values are
 * accumulated in fp64 relative to the channel's value in row 0 (no E[x^2] - E[x]^2 cancellation); per-block partials are
 * merged in a fixed order, so two calls give bit-identical results.  ws: osb_bn_stats_workspace_bytes(n, c) bytes (0 for
 * shapes the call rejects).  Requires n >= 2 (as torch) and c a positive multiple of 32.
 *
 * osb_bn_apply_split: in place, x = act(x * scale + shift + r) with
 *   r = 0                                    res_split == NULL
 *   r = res                                  res_split given, res_scale == res_shift == NULL (BasicBlock identity shortcut)
 *   r = res * res_scale + res_shift          all three given (the downsample branch's raw output with its own statistics)
 *   act = max(., 0) when relu != 0.  res_split has the rows and channels of x and must not alias it. */
size_t osb_bn_stats_workspace_bytes(int64_t n, int32_t c);
int osb_bn_batch_stats(const void *x_split, int64_t n, int32_t c, const float *weight, const float *bias, double eps,
                       double momentum, float *running_mean, float *running_var, int64_t *num_batches_tracked,
                       float *scale, float *shift, void *ws, size_t ws_bytes, void *stream);
int osb_bn_apply_split(void *x_split, int64_t n, int32_t c, const float *scale, const float *shift,
                       const void *res_split, const float *res_scale, const float *res_shift, int32_t relu, void *stream);

/* Training (FusedMinkUNet.forward_train, openscene_b200/engine_train.py; run/distill.py's training step).  The forward keeps what the backward needs:
 *
 * osb_bn_batch_stats_save: osb_bn_batch_stats that also writes the batch mean and invstd = 1 / sqrt(var + eps) (fp32 [c]).
 *   The backward needs them; they cannot be recovered from scale / shift when weight == 0.
 * osb_bn_apply_split_out: osb_bn_apply_split into separate output rows y_split (x_split, the raw convolution output z, is
 *   kept for the backward).  y_split must not overlap x_split or res_split.
 *
 * Backward of y = act(BN(z) + r) given the incoming gradient g (all split rows [n, c]):
 *   g' = g [y > 0] (y_split given: the ReLU mask), or g' = g (y_split NULL: no activation), x^ = (z - mean) invstd
 * osb_bn_backward_reduce: sums = (sum g', sum g' x^) (fp32 [2, c]); dbias = sum g', dweight = sum g' x^ (fp32 [c]),
 *   overwritten, or added to the buffers' values when accumulate != 0.  Sums are taken in fp64 and per-block partials
 *   merged in a fixed order (bit-reproducible, no atomics).  ws: osb_bn_stats_workspace_bytes(n, c) bytes.
 * osb_bn_backward_apply: dz = weight invstd (g' - sums[0] / n - x^ sums[1] / n) into dz_split, with the sums of
 *   osb_bn_backward_reduce.  gp_split (may be NULL) receives g' (gp_accumulate == 0) or gp_split += g': the gradient of the
 *   BasicBlock's identity shortcut.  dz_split and gp_split must not overlap each other or y, g, z. */
int osb_bn_batch_stats_save(const void *x_split, int64_t n, int32_t c, const float *weight, const float *bias, double eps,
                            double momentum, float *running_mean, float *running_var, int64_t *num_batches_tracked,
                            float *scale, float *shift, float *mean, float *invstd, void *ws, size_t ws_bytes, void *stream);
int osb_bn_apply_split_out(const void *x_split, void *y_split, int64_t n, int32_t c, const float *scale, const float *shift,
                           const void *res_split, const float *res_scale, const float *res_shift, int32_t relu, void *stream);
int osb_bn_backward_reduce(const void *y_split, const void *g_split, const void *z_split, int64_t n, int32_t c,
                           const float *mean, const float *invstd, float *sums, float *dweight, float *dbias,
                           int32_t accumulate, void *ws, size_t ws_bytes, void *stream);
int osb_bn_backward_apply(const void *y_split, const void *g_split, const void *z_split, int64_t n, int32_t c,
                          const float *mean, const float *invstd, const float *weight, const float *sums, void *dz_split,
                          void *gp_split, int32_t gp_accumulate, void *stream);

/* Softmax cross-entropy head (FusedMinkUNet.forward_train_ce, openscene_b200/engine_train.py; run/train_mink.py's step):
 * the final 1x1x1 convolution cin -> C of a per-voxel classifier, `CrossEntropyLoss(ignore_index)` over its rows (mean over
 * the labelled rows) and `output.max(1)[1]`, without writing the logits.
 *   x_split      the network's last activation, split rows [n, cin] in internal order; cin a multiple of 32 up to 384
 *   w            fp32 [cin, C], 1 <= C <= 160
 *   row_map      int32 [n]: caller row of internal row r (the coordinate manager's perm, a permutation of 0..n-1);
 *                labels are read and pred written in caller order through it
 *   labels       int32 or int64 [n] (labels_are_i64), caller order; a label outside [0, C) other than ignore_index makes the
 *                loss NaN (callers validate labels first); labels are only read at row_map[r]
 *   ws           osb_ce_head_workspace_bytes(n, cin, C) bytes, 256-byte aligned (0 for shapes the calls reject)
 * osb_ce_head_fwd: z = x w (fp32 accumulation), lse[r] = log sum exp z (fp32 [n], internal order), pred[row_map[r]] = first
 *   argmax of z (int64), n_valid = number of rows whose label != ignore_index (int64 [1]), loss (fp32 [1]) = sum over those
 *   rows of lse - z[label] / n_valid, NaN when n_valid == 0.  The sum is fp64 with per-block partials merged in a fixed order.
 * osb_ce_head_bwd: with g (fp32 [1], the upstream gradient of loss) and n_valid read on the device (no host sync):
 *   d = (softmax(z) - onehot(label)) g / n_valid on labelled rows, 0 elsewhere (z recomputed, softmax = exp(z - lse));
 *   dx_split = d w^T (split rows [n, cin], internal order), dw = sum_r x_r^T d_r (fp32 [cin, C], overwritten).  Every
 *   output is exactly 0 when n_valid == 0.  Partials are merged in a fixed order: two calls give identical bits. */
size_t osb_ce_head_workspace_bytes(int64_t n, int32_t cin, int32_t C);
int osb_ce_head_fwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t C, const int32_t *row_map,
                    const void *labels, int32_t labels_are_i64, int64_t ignore_index, float *lse, int64_t *pred, float *loss,
                    int64_t *n_valid, void *ws, size_t ws_bytes, void *stream);
int osb_ce_head_bwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t C, const int32_t *row_map,
                    const void *labels, int32_t labels_are_i64, int64_t ignore_index, const float *lse, const float *g,
                    const int64_t *n_valid, void *dx_split, float *dw, void *ws, size_t ws_bytes, void *stream);
/* Evaluation head over points (FusedMinkUNet.forward_eval_ce; run/train_mink.py's validate() after the forward): the same
 * row pass as osb_ce_head_fwd, walking points instead of rows.  Point p reads split row row_map[inds_reverse[p]]
 * (row_map[p] when inds_reverse is NULL, then n_pts == n_rows) and its label at p:
 *   row_map      int32 [n_rows]: internal row of caller row v (the coordinate manager's inv_perm)
 *   inds_reverse int64 [n_pts] caller row of every point, values in [0, n_rows), or NULL (may be NULL when n_pts == 0)
 *   labels       int32 or int64 [n_pts] (labels_are_i64); may be NULL when n_pts == 0
 *   loss         fp32 [1] = sum of lse - z[label] over points with a label in [0, C) / their number (fp64 sum, per-block
 *                partials merged in a fixed order); NaN when no point is labelled or n_pts == 0 (torch's 0 / 0)
 *   pred         int64 [n_pts] (may be NULL) = first argmax of z (the first NaN of a row if it holds one)
 *   areas        in/out uint64 [3, C] += intersection | output | target counts of (pred, label), intersectionAndUnionGPU's
 *                rule (util/util.py:132-145): pred is ignored where label == ignore_index, values outside 0..C-1 drop out
 *   bad_labels   in/out int32 [1] += points whose label lies outside [0, C) and is not ignore_index; such a point is left
 *                out of the loss and the counts
 *   ws           osb_ce_head_eval_workspace_bytes(n_pts, cin, C) bytes, 256-byte aligned (0 for shapes the call rejects)
 * Shapes as osb_ce_head_fwd.  No host synchronisation; two calls on the same inputs give the same bits. */
size_t osb_ce_head_eval_workspace_bytes(int64_t n_pts, int32_t cin, int32_t C);
int osb_ce_head_eval(const void *x_split, int64_t n_rows, int32_t cin, const float *w, int32_t C, const int32_t *row_map,
                     const int64_t *inds_reverse, int64_t n_pts, const void *labels, int32_t labels_are_i64,
                     int32_t ignore_index, int64_t *pred, float *loss, uint64_t *areas, int32_t *bad_labels, void *ws,
                     size_t ws_bytes, void *stream);

/* Cosine distillation head on split rows (FusedMinkUNet.forward_train_cosine; run/distill.py's loss_type 'cosine'): the final
 * 1x1x1 layer f = x w, then loss = mean over the m supervised rows of 1 - CosineSimilarity(dim=1, eps=1e-8)(f, t).  The
 * C-wide rows f and their gradient are never written.
 *   x_split  split rows [n, cin] (internal order); cin a multiple of 32 up to 384, C 512 or 768 (other shapes are refused)
 *   w        fp32 [cin, C], 16-byte aligned
 *   rows     int32 [m], 1 <= m <= n: internal row of every supervised row, caller order, distinct (dx is written, not added)
 *   target   fp16 [m, C] in the order of rows, 16-byte aligned; widened to fp32 exactly
 *   state    fp64 [m, 3] = (|f|, f.t, |t|) per supervised row, written by the forward and read by the backward
 *   ws       osb_cos_head_workspace_bytes(m, cin, C) bytes, 256-byte aligned (0 for shapes the calls reject)
 * osb_cos_head_fwd: f = x w (fp32, k ascending), the row sums in fp64; loss (fp32 [1]) = sum_r (1 - f.t / (max(|f|, eps)
 *   max(|t|, eps))) / m, the sum in fp64 with per-block partials merged in a fixed order.
 * osb_cos_head_bwd: with g (fp32 [1], the upstream gradient of loss) read on the device (no host sync), dloss/df_r =
 *   a_r t_r + b_r f_r with a_r = -g / (m n1c n2c), b_r = g (f.t) / (m n1c^2 n2c |f|) (0 when |f| = 0), n1c = max(|f|, eps),
 *   n2c = max(|t|, eps) (torch's clamps, without gradient); dx_split [n, cin] = dloss/df_r w^T at rows[r] and exactly 0 on
 *   every other row; dw (fp32 [cin, C], overwritten) = sum_r x_r^T dloss/df_r.  Every merge is in a fixed order: two calls
 *   give identical bits. */
size_t osb_cos_head_workspace_bytes(int64_t m, int32_t cin, int32_t C);
int osb_cos_head_fwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t C, const int32_t *rows, int64_t m,
                     const void *target, double *state, float *loss, void *ws, size_t ws_bytes, void *stream);
int osb_cos_head_bwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t C, const int32_t *rows, int64_t m,
                     const void *target, const double *state, const float *g, void *dx_split, float *dw, void *ws,
                     size_t ws_bytes, void *stream);

/* L1 distillation head on split rows (FusedMinkUNet.forward_train_l1; run/distill.py's loss_type 'l1'): the final 1x1x1 layer
 * f = x w, then loss = torch.nn.L1Loss()(f, t), the mean of |f - t| over the m x C elements.  The C-wide rows f and their
 * gradient are never written.
 *   x_split  split rows [n, cin] (internal order); cin a multiple of 32 up to 384, C 512 or 768 (other shapes are refused)
 *   w        fp32 [cin, C], 16-byte aligned
 *   rows     int32 [m], 1 <= m <= n: internal row of every supervised row, caller order, distinct (dx is written, not added)
 *   target   fp16 [m, C] in the order of rows, 16-byte aligned; widened to fp32 exactly
 *   signs    uint32 [m, C / 16], 16-byte aligned: sign(f - t) of every element, 2 bits each (element j of a row in bits
 *            2 (j % 16) .. 2 (j % 16) + 1 of word j / 16; 0: d = +-0 or NaN, 1: +1, 2: -1), written by the forward and
 *            the only per-row state the backward reads
 *   ws       osb_l1_head_workspace_bytes(m, cin, C) bytes, 256-byte aligned (0 for shapes the calls reject)
 * osb_l1_head_fwd: f = x w (fp32, k ascending), d = fp32(f - t); loss (fp32 [1]) = fp32(sum |d| / (m C)), the sum in fp64
 *   with per-block partials merged in a fixed order (NaN if any d is NaN, inf if any is infinite).
 * osb_l1_head_bwd: with g (fp32 [1], the upstream gradient of loss) read on the device (no host sync), s = fp32(g * fp32(1 /
 *   fp32(m C))) and dloss/df = s sgn(d) from the signs; dx_split [n, cin] = s (sgn_r w^T) at rows[r] and exactly 0 on every
 *   other row; dw (fp32 [cin, C], overwritten) = s (X^T Sgn), per-split fp32 partials merged in fp64 in a fixed order.  Two
 *   calls give identical bits. */
size_t osb_l1_head_workspace_bytes(int64_t m, int32_t cin, int32_t C);
int osb_l1_head_fwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t C, const int32_t *rows, int64_t m,
                    const void *target, uint32_t *signs, float *loss, void *ws, size_t ws_bytes, void *stream);
int osb_l1_head_bwd(const void *x_split, int64_t n, int32_t cin, const float *w, int32_t C, const int32_t *rows, int64_t m,
                    const uint32_t *signs, const float *g, void *dx_split, float *dw, void *ws, size_t ws_bytes, void *stream);

/* fp32 [n,c] <-> split rows. */
int osb_f32_to_split(const float *in, int64_t n, int32_t c, void *out_split, void *stream);
int osb_split_to_f32(const void *in_split, int64_t n, int32_t c, float *out, void *stream);

/* ------------------------------------------------------ row-wise helpers */
/* out[r,:] = in[idx[r],:]  (fp32 rows of c floats; idx int32) */
int osb_gather_rows_f32(const float *in, const int32_t *idx, int64_t n_out, int32_t c, float *out, void *stream);

/* ------------------------------------------------- open-vocabulary match
 * One pass over the voxel features per query point p (v = inds_reverse[p], or p when NULL):
 *   a = feat[v,:] (fp32 or fp16);  if normalize: a = a / (|a| + 1e-5)
 *   s = fp16( fp16(a) . text[k,:] )  with fp32 accumulation  (text fp16 [K, C] row major)
 *   scores[p,k] = s (fp16, may be NULL), label[p] = argmax_k s (first maximum), smax[p] = max_k s (may be NULL)
 * Mirrors run/evaluate.py:290-292 (distill), :294-296 (fusion), :303-310 (the two normalised products). */
int osb_match_scores(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse,
                     int64_t n_pts, const void *text_f16, int32_t k_text, int32_t normalize, void *scores_f16,
                     int64_t *label, float *smax, void *stream);
/* Ensemble select + final product (run/evaluate.py:316-322):
 *   m = smax3d[p] < smax2d[p];  fe = m ? feat2d_f16[v] : fp16(feat3d[v]);  scores = fe @ text^T;  label = argmax
 *   feat_out_f16 (may be NULL) receives fe. */
int osb_match_ensemble(const float *feat3d, const void *feat2d_f16, int64_t n_vox, int32_t c,
                       const int64_t *inds_reverse, int64_t n_pts, const float *smax3d, const float *smax2d,
                       const void *text_f16, int32_t k_text, void *scores_f16, int64_t *label, void *feat_out_f16,
                       void *stream);

/* Test-time repeat vote (run/evaluate.py:385-425 with test_repeats > 1).  The product of osb_match_scores /
 * osb_match_ensemble (same arguments, same fp16 scores s), and in the same pass, for every point p and column k:
 *   store[p,k] = fp16_rn(store[p,k] + s[p,k])          in/out fp16 [n_pts, K], zero before the first repeat
 *   label_cur[p] = argmax_k s[p,k],  label_acc[p] = argmax_k store[p,k]  (int64, may be NULL)
 * The argmax is torch's CPU `x.float().max(1)[1]`: the first NaN of a row if it holds one, else the first maximum.
 * scores_f16 (may be NULL) receives s bit-identical to osb_match_scores; otherwise s never reaches memory.
 * 1 <= K <= 480.  Store bits are the reference's `store = pred + store` on the CPU applied in repeat order. */
int osb_match_vote(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse,
                   int64_t n_pts, const void *text_f16, int32_t k_text, int32_t normalize, void *scores_f16,
                   void *store_f16, int64_t *label_cur, int64_t *label_acc, void *stream);
int osb_match_ensemble_vote(const float *feat3d, const void *feat2d_f16, int64_t n_vox, int32_t c,
                            const int64_t *inds_reverse, int64_t n_pts, const float *smax3d, const float *smax2d,
                            const void *text_f16, int32_t k_text, void *scores_f16, void *store_f16, int64_t *label_cur,
                            int64_t *label_acc, void *stream);
/* The same vote from a score or logit matrix already in memory (run/eval_mink.py:193-212):
 *   store[p,k] += src[v,k]   v = inds_reverse[p] (or p when NULL, then n_src == n_pts), in the source's precision
 *                            (src_is_f16: fp16 source and store, one fp16 add rounded to nearest even; else fp32)
 *   label_cur / label_acc as above.  1 <= K <= 512. */
int osb_vote_accumulate(const void *src, int32_t src_is_f16, int64_t n_src, const int64_t *inds_reverse, int64_t n_pts,
                        int32_t k, void *store, int64_t *label_cur, int64_t *label_acc, void *stream);

/* Validation tail of run/distill.py (:419-431) in one pass: the product of osb_match_scores with normalize = 0 (same
 * arguments, same fp16 scores s), and for every point p with label y = label[p] (int32 or int64, label_is_i64):
 *   logp   = fp16((s[y] - m) - log(sum_k exp(s[k] - m))) in fp32, m = max_k s[k]  (torch's CUDA log_softmax for Half)
 *   loss   fp16 [1] = fp16(sum of -logp over rows with y != ignore_index / their number), the sum in fp64 with per-block
 *          partials merged in a fixed order; NaN when no row is labelled (torch's `CrossEntropyLoss(ignore_index)`)
 *   pred   int64 [n_pts] (may be NULL) = argmax_k s: the first NaN of a row if it holds one, else the first maximum
 *   areas  in/out uint64 [3, classes] += intersection | output | target counts of (pred, y), intersectionAndUnionGPU's
 *          rule (util/util.py:132-145): pred is ignored where y == ignore_index, values outside 0..classes-1 drop out
 *   bad_labels  in/out int32 [1] += rows whose label lies outside [0, K) and is not ignore_index; such a row is left out
 *          of the loss and the counts
 *   scores_f16 (may be NULL) receives s bit-identical to osb_match_scores; otherwise s never reaches memory.
 *   ws     8-byte aligned workspace of 16 * ceil(n_pts / 128) bytes; ws and label may be NULL when n_pts == 0
 * 1 <= K <= 480, 1 <= classes <= 512.  Two calls on the same inputs give the same bits. */
int osb_match_ce(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse, int64_t n_pts,
                 const void *text_f16, int32_t k_text, const void *label, int32_t label_is_i64, int32_t ignore_index,
                 int32_t classes, void *scores_f16, int64_t *pred, void *loss_f16, uint64_t *areas, int32_t *bad_labels,
                 void *ws, size_t ws_bytes, void *stream);

/* Streaming top-k for vocabularies of any size: the product of osb_match_scores (same arguments, same fp16 scores s, the
 * same bits for every column) over ceil(K / 96) passes, keeping per point p only the topk best columns, best first:
 *   order    NaN above every number (NaNs by ascending column); numbers by descending value, -0 == +0, equal values by
 *            ascending column.  topk = 1 is osb_match_vote's / osb_match_ce's argmax; on rows without NaN it is
 *            osb_match_scores' label, on rows with a NaN it is not (osb_match_scores skips NaN).
 *   label    int64 [n_pts, topk] (required), scores_f16 fp16 [n_pts, topk] (may be NULL): the columns and their scores
 *   smax     fp32 [n_pts] (may be NULL): the largest non-NaN score at its lowest column, -inf when there is none, as
 *            osb_match_scores reports it
 * Nothing of size [n_pts, K] is written.  1 <= K <= OSB_MATCH_TOPK_MAX_TEXT, 1 <= topk <= min(8, K).  Tensor-core route
 * only: OSB_MATCH_SIMT does not apply.  Two calls on the same inputs give the same bits. */
#define OSB_MATCH_TOPK_MAX_TEXT 1048576
int osb_match_topk(const void *feat, int32_t feat_is_f16, int64_t n_vox, int32_t c, const int64_t *inds_reverse,
                   int64_t n_pts, const void *text_f16, int32_t k_text, int32_t normalize, int32_t topk, void *scores_f16,
                   int64_t *label, float *smax, void *stream);
/* The ensemble's final product as a streaming top-k (osb_match_ensemble with the order above):
 *   fe = sel_a[p] < sel_b[p] ? feat2d_f16[v] : fp16(feat3d[v]);  label / scores_f16 = top-k of fe @ text^T
 *   feat_out_f16 (may be NULL) receives fe.  sel_a / sel_b are the smax of two osb_match_topk calls with normalize = 1
 *   (the 3-D and the 2-D features). */
int osb_match_ensemble_topk(const float *feat3d, const void *feat2d_f16, int64_t n_vox, int32_t c,
                            const int64_t *inds_reverse, int64_t n_pts, const float *sel_a, const float *sel_b,
                            const void *text_f16, int32_t k_text, int32_t topk, void *scores_f16, int64_t *label,
                            void *feat_out_f16, void *stream);

/* Scene search (DESIGN.md, "Scene search contract"): fp16 rows [n_rows, c] of scenes stored one after another (scene s
 * owns rows [scene_off[s], scene_off[s+1]); row_scene[r] int32 is the scene of row r) against fp16 queries [nq, c].  The
 * scores are the bits osb_match_scores(rows, feat_is_f16 = 1, normalize = 0, inds_reverse = NULL, text = queries) writes;
 * nothing of size [n_rows, nq] is written.  Order: NaN never ranks, is never a maximum and is never counted; numbers by
 * descending value, -0 == +0; equal values to the lower global row.
 *   top_score_f16 fp16 / top_scene int64 / top_row int64 [nq, k]: the k best rows per query, best first (top_row is the
 *                  row within its scene); slots past the last non-NaN row are (-inf, -1, -1)
 *   scene_max_f16 fp16 / scene_argmax int64 [n_scenes, nq]: the best score of each scene (its own bits) and its row within
 *                  the scene, the lowest on ties; (-inf, -1) when the scene has no non-NaN score
 *   scene_count int64 [n_scenes, nq] (may be NULL; needs threshold, fp32 [nq]): rows with float(s) >= threshold[q]
 * scene_off_host (host memory) and scene_off (device) hold the same n_scenes + 1 offsets; the host copy is checked to
 * run strictly increasing from 0 to n_rows.  1 <= nq <= OSB_SEARCH_MAX_QUERIES, 1 <= k <= OSB_SEARCH_MAX_K,
 * 1 <= n_rows < 2^31; rows and queries 16-byte aligned.  The workspace (osb_search_workspace_bytes, 8-byte aligned,
 * independent of n_rows) is overwritten.  A memset and two launches; two calls on the same inputs give the same bits. */
#define OSB_SEARCH_MAX_QUERIES 96
#define OSB_SEARCH_MAX_K 32
size_t osb_search_workspace_bytes(int64_t n_scenes, int32_t nq, int32_t k);
int osb_search(const void *rows_f16, const int32_t *row_scene, int64_t n_rows, int32_t c, const int64_t *scene_off_host,
               const int64_t *scene_off, int64_t n_scenes, const void *queries_f16, int32_t nq, int32_t k,
               const float *threshold, void *top_score_f16, int64_t *top_scene, int64_t *top_row, void *scene_max_f16,
               int64_t *scene_argmax, int64_t *scene_count, void *ws, size_t ws_bytes, void *stream);

/* Regions of search hits (DESIGN.md, "Region contract").  A hit is a (row, query) with float(s[r, q]) >= threshold[q], s the
 * bits osb_search scores; NaN is never a hit.
 *
 * osb_search_hits: the hit list of one launch of at most OSB_SEARCH_MAX_QUERIES queries, sorted by (query, global row).
 *   scene_count  int64 [n_scenes, nq]: osb_search's counts for the same rows, queries and threshold; n_hits their sum
 *   hit_key      out int64 [n_hits]: (query << 32) | global row, ascending
 *   hit_score_f16 out fp16 [n_hits]: s[row, query]
 *   status       int32, or-ed with OSB_REGIONS_ST_COUNT when a (query, scene) segment does not receive exactly its count
 * Arguments as osb_search; the workspace is osb_search_hits_workspace_bytes (8-byte aligned). */
#define OSB_REGIONS_ST_COUNT 1    /* emitted hits differ from the counts */
#define OSB_REGIONS_ST_RANGE 2    /* a hit's coordinate lies outside |x|, |y|, |z| < 2^17 - 256 */
#define OSB_REGIONS_ST_DUP 4      /* two hits of one (scene, query) share a voxel */
#define OSB_REGIONS_MAX_R 32
size_t osb_search_hits_workspace_bytes(int64_t n_scenes, int32_t nq, int64_t n_hits);
int osb_search_hits(const void *rows_f16, const int32_t *row_scene, int64_t n_rows, int32_t c, const int64_t *scene_off_host,
                    int64_t n_scenes, const void *queries_f16, int32_t nq, const float *threshold,
                    const int64_t *scene_count, int64_t n_hits, int64_t *hit_key, void *hit_score_f16, int32_t *status,
                    void *ws, size_t ws_bytes, void *stream);
/* osb_regions: connected components of the hits of each (scene, query) under Chebyshev distance <= reach (1 or 2) on the
 * int32 coordinates coords [n_rows, 4] = (x, y, z, unused), and the R best per query of those with at least min_voxels
 * voxels, ranked by the search key of their best hit.  n_hits may be 0 (everything padded).
 *   score_f16 fp16 / scene int64 / row int64 / size int64 [nq, R], box_min / box_max int32 [nq, R, 3]: unused slots
 *             (-inf, -1, -1, 0, 0, 0)
 *   n_regions int64 [n_scenes, nq]: regions with at least min_voxels voxels
 *   hit_query / hit_scene / hit_row / hit_region int64 [n_hits] (all four or none): per hit in list order, hit_region the
 *             rank of its region in its query's list or -1
 *   status    or-ed with OSB_REGIONS_ST_RANGE / OSB_REGIONS_ST_DUP (duplicates among hits only)
 * 1 <= nq <= OSB_SEARCH_MAX_QUERIES, 1 <= R <= OSB_REGIONS_MAX_R, min_voxels >= 1; coords 16-byte aligned; the workspace is
 * osb_regions_workspace_bytes (8-byte aligned).  Integer atomics only: two calls give the same bits. */
size_t osb_regions_workspace_bytes(int64_t n_hits);
int osb_regions(const int64_t *hit_key, const void *hit_score_f16, int64_t n_hits, const int32_t *coords,
                const int32_t *row_scene, const int64_t *scene_off, int64_t n_rows, int64_t n_scenes, int32_t nq, int32_t R,
                int32_t reach, int32_t min_voxels, void *score_f16, int64_t *scene, int64_t *row, int64_t *size,
                int32_t *box_min, int32_t *box_max, int64_t *n_regions, int64_t *hit_query, int64_t *hit_scene,
                int64_t *hit_row, int64_t *hit_region, int32_t *status, void *ws, size_t ws_bytes, void *stream);

/* FP8 scene index (DESIGN.md, "FP8 index contract"): each row stored as c e4m3 codes (uint8) and one int8 exponent e, the
 * row it stands for being d = code * 2^e, an exact fp16 row.
 *
 * osb_index_quantize_f8: rows [n, c] (fp16 if rows_are_f16, else fp32, which is rounded to fp16 first) -> codes_out uint8
 *   [n, c] and exp_out int8 [n].  e is the smallest integer with max|h| <= 448 * 2^e, clamped to [-15, 7]; codes are
 *   e4m3(clamp(h * 2^-e, -448, 448)) rounded to nearest even; a row with a NaN or inf element gets NaN codes (0x7f) and
 *   e = 0.  1 <= n < 2^31, rows and codes 16-byte aligned.  One launch, no host synchronisation.
 * osb_search_f8 / osb_search_hits_f8: osb_search / osb_search_hits on the rows d, from codes [n_rows, c] (16-byte aligned)
 *   and row_exp int8 [n_rows]; every output has the bits the fp16 entry point gives on d, with the same workspace. */
int osb_index_quantize_f8(const void *rows, int32_t rows_are_f16, int64_t n, int32_t c, void *codes_out, int8_t *exp_out,
                          void *stream);
int osb_search_f8(const void *codes_f8, const int8_t *row_exp, const int32_t *row_scene, int64_t n_rows, int32_t c,
                  const int64_t *scene_off_host, const int64_t *scene_off, int64_t n_scenes, const void *queries_f16,
                  int32_t nq, int32_t k, const float *threshold, void *top_score_f16, int64_t *top_scene, int64_t *top_row,
                  void *scene_max_f16, int64_t *scene_argmax, int64_t *scene_count, void *ws, size_t ws_bytes,
                  void *stream);
int osb_search_hits_f8(const void *codes_f8, const int8_t *row_exp, const int32_t *row_scene, int64_t n_rows, int32_t c,
                       const int64_t *scene_off_host, int64_t n_scenes, const void *queries_f16, int32_t nq,
                       const float *threshold, const int64_t *scene_count, int64_t n_hits, int64_t *hit_key,
                       void *hit_score_f16, int32_t *status, void *ws, size_t ws_bytes, void *stream);

/* Labelled scene index (DESIGN.md, "Label contract").  row_label int64 / row_label_score fp16 [n_rows] are column 0 of
 * osb_match_topk (topk = 1, normalize = 0, no point expansion) on the index's rows against a vocabulary of k_text classes.
 * A query names m distinct classes classes_host int64 [m] (host memory, each in [0, k_text)); slot j stands for
 * classes_host[j].  A row counts for slot j when its label is classes_host[j] and, with threshold fp32 [m], its label
 * score is not NaN and float(score) >= threshold[j].
 *
 * osb_match_topk_f8: osb_match_topk (inds_reverse = NULL, normalize = 0) over FP8 index rows d = code * 2^e, codes
 *   [n_rows, c] (16-byte aligned) and row_exp int8 [n_rows]; every output has the bits osb_match_topk gives on d.
 * osb_label_counts: counts int64 [n_scenes, m] (overwritten) of the counted rows per scene and slot.  n_scenes * m at most
 *   OSB_LABEL_MAX_COUNTS; threshold may be NULL (every row under its label counts, NaN scores included).  Workspace
 *   osb_label_counts_workspace_bytes (8-byte aligned).
 * osb_label_hits: the hit list of 1 <= m <= OSB_SEARCH_MAX_QUERIES slots in osb_search_hits' layout, which osb_regions
 *   takes: hit_key int64 [n_hits] = (slot << 32) | global row, ascending; hit_score_f16 fp16 [n_hits] the label scores;
 *   counts the osb_label_counts of the same classes and threshold (required), n_hits their sum; status or-ed with
 *   OSB_REGIONS_ST_COUNT when a (slot, scene) segment does not receive exactly its count.  Workspace
 *   osb_label_hits_workspace_bytes (8-byte aligned).
 * Scene offsets are implied by row_scene int32 [n_rows] (non-decreasing, < n_scenes).  Class ids out of range or listed
 * twice are refused on the host.  Integer atomics only: two calls give the same bits; no host synchronisation. */
#define OSB_LABEL_MAX_COUNTS 134217728
int osb_match_topk_f8(const void *codes_f8, const int8_t *row_exp, int64_t n_rows, int32_t c, const void *text_f16,
                      int32_t k_text, int32_t topk, void *scores_f16, int64_t *label, float *smax, void *stream);
size_t osb_label_counts_workspace_bytes(int32_t k_text, int32_t m);
int osb_label_counts(const int64_t *row_label, const void *row_score_f16, const int32_t *row_scene, int64_t n_rows,
                     int64_t n_scenes, int32_t k_text, const int64_t *classes_host, int32_t m, const float *threshold,
                     int64_t *counts, void *ws, size_t ws_bytes, void *stream);
size_t osb_label_hits_workspace_bytes(int32_t k_text, int64_t n_rows, int64_t n_scenes, int32_t m);
int osb_label_hits(const int64_t *row_label, const void *row_score_f16, const int32_t *row_scene, int64_t n_rows,
                   int64_t n_scenes, int32_t k_text, const int64_t *classes_host, int32_t m, const float *threshold,
                   const int64_t *counts, int64_t n_hits, int64_t *hit_key, void *hit_score_f16, int32_t *status, void *ws,
                   size_t ws_bytes, void *stream);

/* Sharded scene index (DESIGN.md, "Sharded index contract"): the per-rank results of osb_search / osb_regions merged into
 * the results of one index holding every scene in ascending global id.  The directory maps each rank's local scene to its
 * global id (scene_gid int64 [n_local]) and each global id to its first global row (row_base int64 [n_global]).
 *
 * osb_shard_keys: a rank's decoded results score_f16 fp16 / scene int64 (local, -1 padding) / row int64 [n] -> key int64
 *   [n]: bits 48-63 the score's order (as osb_search's key: -0 == +0, inf above every finite value), bits 0-47 ~(row_base[g]
 *   + row), 0 for NaN and padding; global_scene int64 [n]: g = scene_gid[scene], -1 for padding.  Refused when the group
 *   holds 2^48 rows or more (n_rows_global).
 * osb_shard_merge: keys int64 [world][nq][m], each [nq][m] list in descending key order -> winners int64 [nq][m]: the
 *   source position w * m + j of the m largest keys per query, largest first (ties among 0 keys to the lower w * m + j).
 *   1 <= world <= OSB_SHARD_MAX_WORLD, 1 <= nq <= OSB_SHARD_MAX_QUERIES, 1 <= m <= OSB_SHARD_MAX_M.
 * osb_shard_hits: the gathered hit lists of one query slice, hit_query (< nq) / hit_grow (global row) / hit_rank (source
 *   rank) / hit_region (rank in the source rank's list, or -1) int64 [n_hits], and the winners int64 [nq][R] of the region
 *   merge -> order int64 [n_hits]: the hits sorted by (query, global row) (a stable radix sort), as source positions;
 *   region_out int64 [n_hits]: per sorted hit the rank of its region in the merged list, -1 when the region is not in it.
 *   The workspace (osb_shard_hits_workspace_bytes, 256-byte aligned) is overwritten.
 * Pointers 8-byte aligned (scores 2).  Integer work only; no host synchronisation. */
#define OSB_SHARD_MAX_WORLD 64
#define OSB_SHARD_MAX_QUERIES 65535
#define OSB_SHARD_MAX_M 32
int osb_shard_keys(const void *score_f16, const int64_t *scene, const int64_t *row, int64_t n, const int64_t *scene_gid,
                   int64_t n_local, const int64_t *row_base, int64_t n_global, int64_t n_rows_global, int64_t *key,
                   int64_t *global_scene, void *stream);
int osb_shard_merge(const int64_t *keys, int32_t world, int32_t nq, int32_t m, int64_t *winners, void *stream);
size_t osb_shard_hits_workspace_bytes(int64_t n_hits);
int osb_shard_hits(const int64_t *hit_query, const int64_t *hit_grow, const int64_t *hit_rank, const int64_t *hit_region,
                   int64_t n_hits, int32_t world, int32_t nq, int32_t R, const int64_t *winners, int64_t *order,
                   int64_t *region_out, void *ws, size_t ws_bytes, void *stream);

/* Optional folded head (engine.forward_scores): rows z = [x L | x U] (fp32, row pitch ld floats) from one 1x1x1
 * convolution with the weights [L | U], W W^T = L L^T, U = W T^T  ->  score_k = fp16((x.U_k) / (|x L| + 1e-5)),
 * label = first argmax.  Same cosine scores as run/evaluate.py:305-310 without materialising the 768-d features. */
int osb_folded_head_finish(const float *z, int64_t n, int32_t ld, int32_t c_norm, int32_t k_text, void *scores_f16,
                           int64_t *label, float *smax, void *stream);

/* ------------------------------------------------------------- voxeliser
 * coords (fp32 or fp64 [n,3]) -> c = floor([p,1] . M^T[:, :3]) with M the HOST 4x4 row-major fp64 matrix,
 * c -= min(c), FNV-64 key (multiply-then-xor over uint64 words), unique by ascending key keeping the
 * FIRST occurrence (np.unique semantics).
 *   coords_vox    out int32 [<=n,3]    voxel coordinates, in ascending-key order
 *   inds          out int64 [<=n]      first-occurrence point index per voxel
 *   inds_reverse  out int64 [n]        voxel row of every point
 *   n_vox_host    out int64 [1] HOST;  min_host out fp64 [3] HOST (the subtracted minimum)
 * SYNC. */
size_t osb_voxelize_workspace_bytes(int64_t n);
int osb_voxelize(const void *coords, int32_t coords_is_f64, int64_t n, const double *matrix_host,
                 int32_t *coords_vox, int64_t *inds, int64_t *inds_reverse, int64_t *n_vox_host,
                 double *min_host, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------- occupancy grid (alternative to the hash table)
 * For a coordinate set whose coordinates are all >= 0 and < (2^nbits << log2_ts): one bit per cell of a 2^nbits cube per
 * batch index, cells in Morton order, + the first row of every 64-cell word.  Because the rows of a set are Morton
 * sorted, row(cell) = first_row[word] + popcount(bits below): a neighbour lookup is two loads from a table of a few
 * MB shared by nearby voxels instead of a probe chain.  Limits: 2 <= nbits <= 9, n_batch << (3 nbits) <= 2^27 cells.
 *   grid        osb_occgrid_bytes(nbits, n_batch) bytes (0 = not representable: use the hash)
 *   coords_int  the set in internal (Morton) order, as produced by osb_coordset_build / _pyramid
 *   status_dev  in/out int32 [1] DEVICE: bit0 set if a coordinate fell outside the grid
 * osb_kernel_map_build_grid / osb_conv_stem_fused_grid are osb_kernel_map_build / osb_conv_stem_fused with the grid of
 * the INPUT set in place of its hash table; results are identical. */
size_t osb_occgrid_bytes(int32_t nbits, int32_t n_batch);
int osb_occgrid_build(const int32_t *coords_int, int64_t n, int32_t log2_ts, int32_t nbits, int32_t n_batch, void *grid,
                      int32_t *status_dev, void *stream);
int osb_kernel_map_build_grid(const int32_t *coords_out, int64_t n_out, const void *grid, int32_t log2_ts, int32_t nbits,
                              int32_t n_batch, int32_t ks_x, int32_t ks_y, int32_t ks_z, int32_t step, int32_t *nbr,
                              int32_t *pairs_per_k, void *stream);
int osb_conv_stem_fused_grid(const float *in, int32_t cin, const int32_t *coords, int64_t n, const void *grid, int32_t log2_ts,
                             int32_t nbits, int32_t n_batch, int32_t ks, int32_t step, const float *w, int32_t cout,
                             const float *scale, const float *shift, int32_t relu, void *out_split, float *out_f32, void *stream);

/* ------------------------------------------------------------- multi-view feature fusion (8f rank 2)
 * One call handles a batch of 1..32 frames, in frame order.
 *   points   fp32 or fp64 [n,3] world coordinates
 *   w2c      fp64 [F,16]  row-major world-to-camera matrices (= inv(pose), fusion_util.py:120)
 *   intr     fp64 [F,4]   (fx, fy, cx, cy) per frame (intrinsic[0][0], [1][1], [0][2], [1][2])
 *   depth    fp64 [F,H,W] metres, or NULL (then the test is p_z > 0, fusion_util.py:134)
 *   feat     fp16 [F,H,W,C] per-pixel features (the memory the reference holds as a permuted [C,H,W] view),
 *            C % 8 == 0, C <= 1024
 *   sum      in/out fp32 [n,C]; counter in/out fp32 [n]: sum += feature, counter += 1 for every frame that sees the
 *            point, applied in frame order (bit-identical to the reference's per-frame fp32 adds).
 *            sum == NULL computes the mapping only.
 *   mapping  out int32 [F,n,3] = (row v, col u, visible) as compute_mapping returns it, or NULL
 *   ws       osb_fusion_workspace_bytes(n, F) bytes */
size_t osb_fusion_workspace_bytes(int64_t n, int32_t n_frames);
int osb_fusion_accumulate(const void *points, int32_t points_is_f64, int64_t n, const double *w2c, const double *intr,
                          const double *depth, const void *feat, int32_t n_frames, int32_t H, int32_t W, int32_t C,
                          int32_t cut_bound, double vis_thres, float *sum, float *counter, int32_t *mapping, void *ws,
                          size_t ws_bytes, void *stream);
/* feat_bank = sum / (counter == 0 ? 1e-5 : counter)   (scannet_openseg.py:104-105); feat_bank may alias sum */
int osb_fusion_finalize(const float *sum, const float *counter, int64_t n, int32_t C, float *feat_bank, void *stream);

/* ------------------------------------------------------------- segmentation metrics (8f rank 4)
 * confusion  in/out uint64 [(C+1),(C+1)], rows = prediction, columns = ground truth; points with gt == ignore_id are
 *            skipped, predictions equal to nofeat_id land in row C (util/metric.py:13-20; the caller slices [:C,:C]).
 * bad_labels in/out int32 [1]: number of labels outside the valid range (the reference would raise in reshape).
 * Labels are int32 or int64 device arrays. */
int osb_confusion_accumulate(const void *pred, const void *gt, int32_t labels_are_i64, int64_t n, int32_t num_classes,
                             int32_t ignore_id, int32_t nofeat_id, uint64_t *confusion, int32_t *bad_labels, void *stream);
/* areas in/out uint64 [3,K] = (intersection, output area, target area) with the reference's histc semantics
 * (util/util.py:132-145): where target == ignore_id the prediction is ignored too; labels outside 0..K-1 are dropped.
 * union = output + target - intersection. */
int osb_intersection_union(const void *output, const void *target, int32_t labels_are_i64, int64_t n, int32_t K,
                           int32_t ignore_id, uint64_t *areas, void *stream);

/* ------------------------------------------------------------- fused-feature remap after voxelisation (8f rank 3)
 * The fused 2-D features of a scene are stored as {feat [M,C], mask_full bool [n_pts]} with one feat row per True
 * entry of mask_full, in point order (scripts/feature_fusion/fusion_util.py:87-89).  Given the voxeliser's
 * representative point per voxel (vox_ind), produce what dataset/feature_loader.py:101-172 hands to the model:
 *   mask_vox  out uint8 [n_vox]            mask_full[vox_ind]                                  (:127)
 *   feat_out  out [<= n_vox, row_bytes]    keep_all == 0 (train): rows of the voxels with mask_vox set, in voxel
 *                                          order (:128-145); keep_all != 0 (val / test): one row per voxel, zeros
 *                                          where the voxel has no feature (:107-111,167-170)
 *   n_out_host out int64 [1] HOST          rows written
 * Rows are opaque: row_bytes = C * element size, a multiple of 16.  m_rows must equal popcount(mask_full).  SYNC. */
size_t osb_feature_remap_workspace_bytes(int64_t n_pts, int64_t n_vox);
int osb_feature_remap(const uint8_t *mask_full, int64_t n_pts, const int64_t *vox_ind, int64_t n_vox, const void *feat,
                      int64_t m_rows, int32_t row_bytes, int32_t keep_all, uint8_t *mask_vox, void *feat_out,
                      int64_t *n_out_host, void *ws, size_t ws_bytes, void *stream);

/* ------------------------------------------------------------- training augmentation (dataset/augmentation.py)
 * The random draws stay on the host in the reference's order; these calls do the per-point / per-voxel arithmetic with
 * NumPy's rounding, bit for bit.  dtype codes: 0 fp32, 1 fp64, 2 int32.  None of them synchronises.
 *   osb_aug_minmax        minmax out fp64 [2c] DEVICE = column minima then maxima of x [n,c] (rows != NULL: of
 *                         x[rows[i]]), NaN-propagating like np.min / np.max; 1 <= c <= 4;
 *                         ws osb_aug_minmax_workspace_bytes(c) bytes
 *   osb_aug_blur          in place on grid fp32 [X,Y,Z,ch]: ElasticDistortion's smoothing = scipy.ndimage.convolve with
 *                         the float32(1/3) 3-tap box along x, y, z, twice, mode='constant' (double accumulation over
 *                         taps -1, 0, +1 from 0.0, one rounding to fp32 per pass); tmp is scratch of the same size
 *   osb_aug_elastic_interp out fp64 [n,3] = p + RegularGridInterpolator(axes, noise, bounds_error=0, fill_value=0)(p)
 *                         * magnitude for pts fp32 / fp64 [n,3], noise fp32 [X,Y,Z,3], axes fp64 [X+Y+Z] DEVICE
 *   osb_aug_input_transforms  one pass over n voxels (feats / labels read at rows[v] when rows != NULL):
 *                         stages OSB_AUG_*; params_host fp64 [8] = (1 - blend, blend, tr[3], jitter_std * 255, hue,
 *                         saturation ratio); coords_max fp64 [3] DEVICE (for the flips), feats_minmax fp64 [6] DEVICE
 *                         (auto-contrast), jitter fp64 [n,3] DEVICE raw standard normals.  Outputs, any may be NULL:
 *                         coords_out / feats_out [n,3] in the input types; item_coords int32 [n,4] = (batch_index,
 *                         x, y, z); item_feats fp32 [n,3] (float(f) / 127.5 - 1 with OSB_AUG_INPUT_COLOR, else 1);
 *                         item_labels int64 [n]. */
#define OSB_AUG_FLIP_X 1
#define OSB_AUG_FLIP_Y 2
#define OSB_AUG_AUTOCONTRAST 4
#define OSB_AUG_TRANSLATE 8
#define OSB_AUG_JITTER 16
#define OSB_AUG_HUE_SAT 32
#define OSB_AUG_INPUT_COLOR 64
#define OSB_AUG_ALL 127
size_t osb_aug_minmax_workspace_bytes(int32_t c);
int osb_aug_minmax(const void *x, int32_t dtype, const int64_t *rows, int64_t n, int32_t c, double *minmax, void *ws,
                   size_t ws_bytes, void *stream);
int osb_aug_blur(float *grid, float *tmp, int32_t X, int32_t Y, int32_t Z, int32_t ch, void *stream);
int osb_aug_elastic_interp(const void *pts, int32_t pts_is_f64, int64_t n, const float *noise, int32_t X, int32_t Y,
                           int32_t Z, const double *axes, double magnitude, double *out, void *stream);
int osb_aug_input_transforms(const void *coords, int32_t coords_dtype, const void *feats, int32_t feats_is_f64,
                             const uint8_t *labels, const int64_t *rows, int64_t n, const double *coords_max,
                             const double *feats_minmax, const double *jitter, const double *params_host, int32_t stages,
                             int32_t batch_index, void *coords_out, void *feats_out, int32_t *item_coords,
                             float *item_feats, int64_t *item_labels, void *stream);

/* ---- optimiser step and in-place weight re-pack (csrc/optim.cu) ------------------------------------------------------
 * Multi-tensor updates: one launch over a DEVICE table of tensors, every tensor cut into chunks of chunk_elems elements
 * (a multiple of 4); chunk_begin = the table's running sum of ceil(numel / chunk_elems), n_chunks its total.  fp32,
 * element-wise, in the order of operations of torch.optim's foreach implementations (_multi_tensor_adam / _sgd), each
 * rounding spelled out (DESIGN.md "Optimiser contract"):
 *   osb_optim_adam   m = lerp(m, g, lerp_w); v = v * beta2 + one_minus_beta2 * (g * g);
 *                    p = p + step_size * (m / (sqrt(v) / bc2_sqrt + eps))
 *   osb_optim_sgd    d = g + weight_decay * p (weight_decay != 0); with a momentum buffer b: b = d if first else
 *                    b * momentum + d, then d = b; p = p + neg_lr * d
 *   osb_conv_repack  every job writes the split-bf16 operand osb_conv_pack_weights would make ([K, cout_pad, cin] rows,
 *                    weight element (k, n, c) read at w[k sk + n sn + c sc]) into an existing buffer; chunks over
 *                    K * cout_pad * cin packed elements per job.
 * osb_optim_entry_bytes(kind): the size of one table entry (0 Adam, 1 SGD, 2 re-pack job; 0 for any other kind). */
typedef struct osb_adam_tensor {
  float *param;
  const float *grad;
  float *exp_avg;
  float *exp_avg_sq;
  int64_t numel;
  int64_t chunk_begin;
  float step_size;          /* -(lr / (1 - beta1^t)), in double then rounded once */
  float bc2_sqrt;           /* (1 - beta2^t)^0.5, in double then rounded once */
  float lerp_w;             /* 1 - beta1 */
  float beta2;
  float one_minus_beta2;
  float eps;
} osb_adam_tensor;
typedef struct osb_sgd_tensor {
  float *param;
  const float *grad;
  float *momentum_buffer;   /* NULL: momentum 0 */
  int64_t numel;
  int64_t chunk_begin;
  float neg_lr;
  float weight_decay;
  float momentum;
  int32_t first;            /* the buffer is new: b = d (torch's clone) */
} osb_sgd_tensor;
typedef struct osb_pack_job {
  const float *w;
  void *wpack;
  int64_t sk, sn, sc;
  int64_t chunk_begin;
  int32_t K, cin, cout, cout_pad;
} osb_pack_job;
size_t osb_optim_entry_bytes(int32_t kind);
int osb_optim_adam(const osb_adam_tensor *table, int32_t n_tensors, int64_t chunk_elems, int64_t n_chunks, void *stream);
int osb_optim_sgd(const osb_sgd_tensor *table, int32_t n_tensors, int64_t chunk_elems, int64_t n_chunks, void *stream);
int osb_conv_repack(const osb_pack_job *jobs, int32_t n_jobs, int64_t chunk_elems, int64_t n_chunks, void *stream);

/* ------------------------------------------------------------------ pooling (fp32, CUDA cores)
 * `MinkowskiSumPooling` / `MinkowskiAvgPooling` / `MinkowskiMaxPooling` (models/resnet_base.py:54) and the global poolings
 * (:68).  mode: 0 sum, 1 avg, 2 max.  No atomics: two runs give the same bits.
 *   osb_pool_fwd   out[o] over the present offsets k of nbr[K][n_out] (input row nbr[k][o], -1 none), ascending k:
 *                  sum = fp32 adds from +0.0; avg = sum / fp32(max(count, 1)) and count[o] (int32) written;
 *                  max = the largest input, first NaN wins, ties (+-0 equal) to the lowest k, 0 when no offset is present;
 *                  argk[o, c] (uint16) = the winning k, 0xFFFF for none.  1 <= K <= 65535.
 *   osb_pool_bwd   on the transposed map nbr_t[K][n_in]: gin[i] = fp32 adds over ascending k of, with o = nbr_t[k][i]:
 *                  g[o] (sum), fp32(g[o] / max(count[o], 1)) (avg), g[o, c] where argk[o, c] == k (max).
 *   osb_global_pool_fwd  out[b, c] over the rows r with batch[r] == b, rows in the caller's order, 1 <= n_batch:
 *                  sum / avg: fp64 partials per chunk of rows, merged in chunk order and rounded to fp32 once (avg divides
 *                  by the row count in fp64 first; count[b] written); an empty batch gives 0 (sum) or NaN (avg);
 *                  max: exact, first NaN wins, ties to the lowest row, argrow[b, c] = the winning row; empty: -inf, -1.
 *                  The workspace (osb_global_pool_workspace_bytes, 16-byte aligned) is overwritten.
 *   osb_global_pool_bwd  gin[r] = g[batch[r]] (sum), fp32(g[b] / count[b]) (avg), g[b, c] on the winning row else 0 (max).
 * count is needed for avg, argk / argrow for max; both are ignored (may be NULL) in the other modes. */
int osb_pool_fwd(const float *in, int32_t c, const int32_t *nbr, int64_t n_out, int32_t K, int32_t mode, float *out,
                 int32_t *count, uint16_t *argk, void *stream);
int osb_pool_bwd(const float *gout, int32_t c, const int32_t *nbr_t, int64_t n_in, int32_t K, int32_t mode,
                 const int32_t *count, const uint16_t *argk, float *gin, void *stream);
size_t osb_global_pool_workspace_bytes(int64_t n, int32_t c, int32_t n_batch);
int osb_global_pool_fwd(const float *in, const int32_t *batch, int64_t n, int32_t c, int32_t n_batch, int32_t mode,
                        float *out, int32_t *count, int32_t *argrow, void *ws, size_t ws_bytes, void *stream);
int osb_global_pool_bwd(const float *gout, const int32_t *batch, int64_t n, int32_t c, int32_t mode, const int32_t *count,
                        const int32_t *argrow, float *gin, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* OSB200_H */
