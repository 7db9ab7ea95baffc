// Stem convolution (conv0p1s1: 5x5x5, 3 -> 32; models/mink_unet.py:47-48) with the kernel-map probe
// fused in.  One warp per output voxel: each round 32 lanes probe 32 of the 125 offsets in the
// coordinate hash and, on a hit, fetch the neighbour's (<= 3) input features; the hits are compacted
// with a ballot into shared memory as float4(x0, x1, x2, offset); then lane n accumulates output
// channel n with one broadcast LDS.128 (the hit) and one LDS.128 (W[k][:, n]) per hit.
// The 5^3 map (500 B / voxel) is never written to HBM.  fp32 FMA; BatchNorm(eval)+ReLU folded.
#include "common.cuh"
#include <algorithm>

namespace osb {

constexpr int STEM_WARPS = 16;

// neighbour lookup: coordinate hash (one 64-bit add per neighbour key) or occupancy grid (common.cuh)
struct StemHashLookup {
  const HashSlot *slots;
  uint64_t mask;
  __device__ int operator()(const int4 &c, uint64_t base, unsigned long long dk) const { return hash_lookup(slots, mask, base + dk); }
};
struct StemGridLookup {
  OccGridView g;
  __device__ int operator()(const int4 &c, uint64_t, unsigned long long dk) const {
    // pack_delta stores the three signed deltas in 18-bit fields of one sum; undo it field by field
    const long long d = (long long)dk;
    const int dx = (int)((long long)((unsigned long long)d << 46) >> 46);
    const long long r1 = (d - dx) >> 18;
    const int dy = (int)((long long)((unsigned long long)r1 << 46) >> 46);
    const int dz = (int)((r1 - dy) >> 18);
    return occgrid_lookup(g, c.x, c.y + dx, c.z + dy, c.w + dz);
  }
};

template <typename Lookup>
__global__ void __launch_bounds__(STEM_WARPS * 32)
k_conv_stem(const float *__restrict__ in, int cin, const int4 *__restrict__ coords, int64_t n,
            const Lookup lookup, int ks, int step, const float *__restrict__ w, int cout,
            const float *__restrict__ scale, const float *__restrict__ shift, int relu, uint8_t *__restrict__ out_split,
            float *__restrict__ out_f32) {
  extern __shared__ float4 s_w4[];                     // [K][32]: (W[k][0][n], W[k][1][n], W[k][2][n], 0)
  __shared__ float4 s_hit[STEM_WARPS][32];
  __shared__ unsigned long long s_dk[352];             // packed key delta of every offset (no div/mod in the probe loop)
  const int K = ks * ks * ks;
  for (int e = threadIdx.x; e < K * 32; e += blockDim.x) {
    const int k = e >> 5, nn = e & 31;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (nn < cout) {
      v.x = __ldg(w + ((int64_t)k * cin + 0) * cout + nn);
      if (cin > 1) v.y = __ldg(w + ((int64_t)k * cin + 1) * cout + nn);
      if (cin > 2) v.z = __ldg(w + ((int64_t)k * cin + 2) * cout + nn);
    }
    s_w4[e] = v;
  }
  const int half = ks / 2;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int ix = k % ks, iy = (k / ks) % ks, iz = k / (ks * ks);
    const int dx = ((ks & 1) ? ix - half : ix) * step, dy = ((ks & 1) ? iy - half : iy) * step,
              dz = ((ks & 1) ? iz - half : iz) * step;
    s_dk[k] = pack_delta(dx, dy, dz);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float sc = (scale && lane < cout) ? __ldg(scale + lane) : 1.f;
  const float sh = (shift && lane < cout) ? __ldg(shift + lane) : 0.f;
  const int64_t warps_total = (int64_t)gridDim.x * STEM_WARPS;
  for (int64_t o = (int64_t)blockIdx.x * STEM_WARPS + warp; o < n; o += warps_total) {
    const int4 c = __ldg(coords + o);
    const uint64_t base = pack_key(c.x, c.y, c.z, c.w);
    float acc = 0.f;
    for (int kb = 0; kb < K; kb += 32) {
      const int k = kb + lane;
      int row = -1;
      if (k < K) row = lookup(c, base, s_dk[k]);
      float4 h = make_float4(0.f, 0.f, 0.f, __int_as_float(k));
      if (row >= 0) {
        const float *xp = in + (int64_t)row * cin;
        h.x = __ldg(xp);
        if (cin > 1) h.y = __ldg(xp + 1);
        if (cin > 2) h.z = __ldg(xp + 2);
      }
      const unsigned bal = __ballot_sync(0xffffffffu, row >= 0);
      if (row >= 0) s_hit[warp][__popc(bal & ((1u << lane) - 1))] = h;
      __syncwarp();
      const int nhit = __popc(bal);
#pragma unroll 4
      for (int j = 0; j < nhit; ++j) {
        const float4 hv = s_hit[warp][j];                               // broadcast
        const float4 wv = s_w4[(__float_as_int(hv.w) << 5) + lane];     // conflict-free
        acc = fmaf(hv.x, wv.x, acc);
        acc = fmaf(hv.y, wv.y, acc);
        acc = fmaf(hv.z, wv.z, acc);
      }
      __syncwarp();
    }
    if (lane < cout) {
      float y = fmaf(acc, sc, sh);
      if (relu) y = fmaxf(y, 0.f);
      if (out_split) {
        __nv_bfloat16 hi, lo;
        split_bf16(y, hi, lo);
        uint8_t *p = out_split + o * (int64_t)cout * 4 + split_off_hi(lane);
        *reinterpret_cast<__nv_bfloat16 *>(p) = hi;
        *reinterpret_cast<__nv_bfloat16 *>(p + 64) = lo;
      }
      if (out_f32) out_f32[o * cout + lane] = y;
    }
  }
}

}  // namespace osb

using namespace osb;

extern "C" {

static int stem_check(int32_t cin, int32_t cout, int32_t ks, const void *out_split, const float *scale, const float *shift, int64_t n,
                      size_t *smem_out) {
  const int K = ks * ks * ks;
  OSB_CHECK(cin >= 1 && cin <= 3 && cout >= 1 && cout <= 32, "osb_conv_stem_fused: needs cin <= 3, cout <= 32 (got %d, %d)", cin, cout);
  OSB_CHECK(K >= 1 && K <= 343, "osb_conv_stem_fused: kernel volume %d not supported", K);
  OSB_CHECK(out_split == nullptr || cout == 32, "osb_conv_stem_fused: split output needs cout == 32");
  OSB_CHECK((scale == nullptr) == (shift == nullptr), "osb_conv_stem_fused: scale and shift go together");
  OSB_CHECK(n > 0, "osb_conv_stem_fused: bad n");
  *smem_out = (size_t)K * 32 * sizeof(float4);
  OSB_CHECK(*smem_out <= 200 * 1024, "osb_conv_stem_fused: weights do not fit in shared memory");
  return 0;
}

int osb_conv_stem_fused(const float *in, int32_t cin, const int32_t *coords, int64_t n, const void *slots, int64_t cap,
                        int32_t ks, int32_t step, const float *w, int32_t cout, const float *scale, const float *shift,
                        int32_t relu, void *out_split, float *out_f32, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  size_t smem = 0;
  if (stem_check(cin, cout, ks, out_split, scale, shift, n, &smem)) return 1;
  OSB_CHECK(slots != nullptr && cap > 0 && (cap & (cap - 1)) == 0, "osb_conv_stem_fused: bad hash table");
  OSB_SMEM_ATTR_ONCE(k_conv_stem<StemHashLookup>, 200 * 1024);
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n, STEM_WARPS), 132 * 3);
  const StemHashLookup lk{(const HashSlot *)slots, (uint64_t)cap - 1};
  k_conv_stem<StemHashLookup><<<grid, STEM_WARPS * 32, smem, stream>>>(in, cin, (const int4 *)coords, n, lk, ks, step, w, cout, scale,
                                                                       shift, relu, (uint8_t *)out_split, out_f32);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_conv_stem_fused_grid(const float *in, int32_t cin, const int32_t *coords, int64_t n, const void *grid_, int32_t log2_ts,
                             int32_t nbits, int32_t n_batch, int32_t ks, int32_t step, const float *w, int32_t cout,
                             const float *scale, const float *shift, int32_t relu, void *out_split, float *out_f32, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  size_t smem = 0;
  if (stem_check(cin, cout, ks, out_split, scale, shift, n, &smem)) return 1;
  OSB_CHECK(grid_ != nullptr && nbits >= 2 && nbits <= 9 && log2_ts >= 0 && log2_ts <= 16 && n_batch >= 1 && n_batch <= 1024 &&
                (int64_t)n_batch * occgrid_words_per_batch(nbits) <= ((int64_t)1 << 21),
            "osb_conv_stem_fused_grid: bad occupancy grid (nbits %d, log2_ts %d, n_batch %d)", nbits, log2_ts, n_batch);
  OSB_CHECK(ks * step < (1 << 16), "osb_conv_stem_fused_grid: offsets too large");
  OSB_SMEM_ATTR_ONCE(k_conv_stem<StemGridLookup>, 200 * 1024);
  const int64_t words = (int64_t)n_batch * occgrid_words_per_batch(nbits);
  StemGridLookup lk;
  lk.g.bitmap = reinterpret_cast<const unsigned long long *>(grid_);
  lk.g.first_row = reinterpret_cast<const int32_t *>(reinterpret_cast<const unsigned long long *>(grid_) + words);
  lk.g.nbits = nbits; lk.g.log2_ts = log2_ts; lk.g.n_batch = n_batch;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(n, STEM_WARPS), 132 * 3);
  k_conv_stem<StemGridLookup><<<grid, STEM_WARPS * 32, smem, stream>>>(in, cin, (const int4 *)coords, n, lk, ks, step, w, cout, scale,
                                                                       shift, relu, (uint8_t *)out_split, out_f32);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
