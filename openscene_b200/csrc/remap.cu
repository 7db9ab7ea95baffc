// Fused-feature remap after voxelisation (SURVEY.md 8f rank 3, the loader side): the fused 2-D features are stored as
// {feat [M,C] (rows of the True points of mask_full, in point order), mask_full bool [N_pts]}
// (scripts/feature_fusion/fusion_util.py:87-89); after voxelisation the loader needs, per voxel, whether its
// representative point has a feature and that feature row (dataset/feature_loader.py:101-172).  The reference does it
// with nonzero / cumsum / three index passes on the CPU; here: two scans and one row-gather kernel.
#include "common.cuh"

#include "sortscan.cuh"
#include <algorithm>

namespace osb {

__global__ void k_remap_flags_pts(const uint8_t *__restrict__ mask_full, int64_t n, int32_t *__restrict__ flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flag[i] = mask_full[i] ? 1 : 0;
}

__global__ void k_remap_flags_vox(const uint8_t *__restrict__ mask_full, int64_t n_pts, const int64_t *__restrict__ vox_ind, int64_t n_vox,
                                  uint8_t *__restrict__ mask_vox, int32_t *__restrict__ flag, int32_t *__restrict__ bad) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_vox) return;
  const int64_t p = vox_ind[j];
  uint8_t m = 0;
  if (p < 0 || p >= n_pts) atomicAdd(bad, 1);
  else m = mask_full[p] ? 1 : 0;
  mask_vox[j] = m;                                      // feature_loader.py:127  mask = mask_chunk[vox_ind]
  flag[j] = m;
}

// warp per voxel; rows are row_bytes (multiple of 16) long
__global__ void __launch_bounds__(256)
k_remap_rows(const int64_t *__restrict__ vox_ind, int64_t n_vox, const uint8_t *__restrict__ mask_vox, const int32_t *__restrict__ rank1,
             const int32_t *__restrict__ pos1, const uint8_t *__restrict__ feat, int row_bytes, int keep_all, uint8_t *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int chunks = row_bytes / 16;
  for (int64_t j = warp0; j < n_vox; j += n_warps) {
    const bool has = mask_vox[j] != 0;
    if (!has && !keep_all) continue;
    const int64_t dst = keep_all ? j : (int64_t)pos1[j] - 1;          // feature_loader.py:133-142: rows in voxel order
    uint4 *o = reinterpret_cast<uint4 *>(out + dst * row_bytes);
    if (has) {
      const int64_t src = (int64_t)rank1[vox_ind[j]] - 1;              // index3[chunk_ind] - 1
      const uint4 *s = reinterpret_cast<const uint4 *>(feat + src * row_bytes);
      for (int c = lane; c < chunks; c += 32) o[c] = __ldg(s + c);
    } else {
      for (int c = lane; c < chunks; c += 32) o[c] = make_uint4(0, 0, 0, 0);   // :108-110 zeros where no feature (val / test)
    }
  }
}

}  // namespace osb

using namespace osb;

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

extern "C" {

size_t osb_feature_remap_workspace_bytes(int64_t n_pts, int64_t n_vox) {
  const int64_t m = std::max<int64_t>(std::max(n_pts, n_vox), 1);
  return 2 * align256((size_t)std::max<int64_t>(n_pts, 1) * 4) + 2 * align256((size_t)std::max<int64_t>(n_vox, 1) * 4) +
         align256(scan_ws_bytes(m)) + 256;
}

int osb_feature_remap(const uint8_t *mask_full, int64_t n_pts, const int64_t *vox_ind, int64_t n_vox, const void *feat,
                      int64_t m_rows, int32_t row_bytes, int32_t keep_all, uint8_t *mask_vox, void *feat_out,
                      int64_t *n_out_host, void *ws, size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n_pts > 0 && n_pts < (1ll << 31) && n_vox >= 0 && n_vox <= n_pts, "osb_feature_remap: sizes out of range (n_pts %lld, n_vox %lld)",
            (long long)n_pts, (long long)n_vox);
  OSB_CHECK(row_bytes > 0 && row_bytes % 16 == 0, "osb_feature_remap: row size %d bytes must be a multiple of 16", row_bytes);
  OSB_CHECK(ws_bytes >= osb_feature_remap_workspace_bytes(n_pts, n_vox), "osb_feature_remap: workspace too small");
  OSB_CHECK(n_out_host != nullptr, "osb_feature_remap: n_out_host is null");
  *n_out_host = 0;
  if (n_vox == 0) return 0;
  uint8_t *w = reinterpret_cast<uint8_t *>(ws);
  int32_t *flag_p = reinterpret_cast<int32_t *>(w); w += align256((size_t)n_pts * 4);
  int32_t *rank1 = reinterpret_cast<int32_t *>(w); w += align256((size_t)n_pts * 4);
  int32_t *flag_v = reinterpret_cast<int32_t *>(w); w += align256((size_t)n_vox * 4);
  int32_t *pos1 = reinterpret_cast<int32_t *>(w); w += align256((size_t)n_vox * 4);
  void *scan_ws = w; w += align256(scan_ws_bytes(std::max(n_pts, n_vox)));
  int32_t *bad = reinterpret_cast<int32_t *>(w);
  OSB_CUDA(cudaMemsetAsync(bad, 0, 4, stream));
  k_remap_flags_pts<<<(unsigned)ceil_div(n_pts, 256), 256, 0, stream>>>(mask_full, n_pts, flag_p);
  OSB_LAUNCH_CHECK();
  OSB_CHECK(inclusive_scan_i32(flag_p, rank1, n_pts, scan_ws, stream) == 0, "osb_feature_remap: scan launch failed");
  k_remap_flags_vox<<<(unsigned)ceil_div(n_vox, 256), 256, 0, stream>>>(mask_full, n_pts, vox_ind, n_vox, mask_vox, flag_v, bad);
  OSB_LAUNCH_CHECK();
  OSB_CHECK(inclusive_scan_i32(flag_v, pos1, n_vox, scan_ws, stream) == 0, "osb_feature_remap: scan launch failed");
  int32_t h[3] = {0, 0, 0};     // popcount(mask_full), rows kept, bad indices
  OSB_CUDA(cudaMemcpyAsync(&h[0], rank1 + (n_pts - 1), 4, cudaMemcpyDeviceToHost, stream));
  OSB_CUDA(cudaMemcpyAsync(&h[1], pos1 + (n_vox - 1), 4, cudaMemcpyDeviceToHost, stream));
  OSB_CUDA(cudaMemcpyAsync(&h[2], bad, 4, cudaMemcpyDeviceToHost, stream));
  OSB_CUDA(cudaStreamSynchronize(stream));
  OSB_CHECK(h[2] == 0, "osb_feature_remap: %d voxel indices outside 0..n_pts-1", h[2]);
  OSB_CHECK((int64_t)h[0] == m_rows, "osb_feature_remap: feat has %lld rows but mask_full has %d True entries", (long long)m_rows, h[0]);
  const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div(n_vox, 8), 132 * 16);
  k_remap_rows<<<blocks, 256, 0, stream>>>(vox_ind, n_vox, mask_vox, rank1, pos1, (const uint8_t *)feat, row_bytes, keep_all, (uint8_t *)feat_out);
  OSB_LAUNCH_CHECK();
  *n_out_host = keep_all ? n_vox : (int64_t)h[1];
  return 0;
}

}  // extern "C"
