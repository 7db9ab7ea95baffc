// Training-time augmentation of dataset/augmentation.py on the device, bit for bit.  The random draws stay on the host
// (Python `random` / `np.random`, same calls and order as the reference); these kernels do the O(points) and O(voxels)
// arithmetic the draws drive:
//   osb_aug_minmax            exact column min / max (NaN-propagating like np.min / np.max)
//   osb_aug_blur              ElasticDistortion's smoothing: scipy.ndimage.convolve with the 3-tap 1/3 box along x, y, z,
//                             twice, constant-0 borders (augmentation.py:171-184)
//   osb_aug_elastic_interp    RegularGridInterpolator(ax, noise, bounds_error=0, fill_value=0)(p) * magnitude + p
//   osb_aug_input_transforms  RandomHorizontalFlip, ChromaticAutoContrast, ChromaticTranslation, ChromaticJitter and
//                             HueSaturationTranslation in one pass, plus the loader's coords / feats / labels outputs
// The build contracts a*b+c into FMAs, so every rounding step here is spelled out with __dmul_rn / __dadd_rn / ... to
// keep NumPy's one-rounding-per-operation order.
#include "common.cuh"

#include <algorithm>
#include <type_traits>

namespace osb {

static constexpr int kMinmaxBlocks = 256;
static constexpr int kMinmaxMaxCols = 4;

enum : int32_t { AUG_F32 = 0, AUG_F64 = 1, AUG_I32 = 2 };

// np.minimum / np.maximum: a NaN on either side wins
__device__ __forceinline__ double nan_min(double a, double b) { return (a != a || a < b) ? a : b; }
__device__ __forceinline__ double nan_max(double a, double b) { return (a != a || a > b) ? a : b; }

template <typename T>
__device__ __forceinline__ double load_d(const T *p, int64_t i) { return (double)p[i]; }

template <typename T, int c>
__global__ void k_aug_minmax_partial(const T *__restrict__ x, const int64_t *__restrict__ rows, int64_t n,
                                     double *__restrict__ part) {
  double mn[c], mx[c];
  bool any = false;
#pragma unroll
  for (int j = 0; j < c; ++j) { mn[j] = 0.0; mx[j] = 0.0; }
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = rows ? rows[i] : i;
#pragma unroll
    for (int j = 0; j < c; ++j) {
      const double v = load_d(x, r * c + j);
      mn[j] = any ? nan_min(mn[j], v) : v;
      mx[j] = any ? nan_max(mx[j], v) : v;
    }
    any = true;
  }
  __shared__ double s_mn[c][256], s_mx[c][256];
  __shared__ int s_any[256];
#pragma unroll
  for (int j = 0; j < c; ++j) { s_mn[j][threadIdx.x] = mn[j]; s_mx[j][threadIdx.x] = mx[j]; }
  s_any[threadIdx.x] = any;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      const int o = threadIdx.x + s;
      if (s_any[o]) {
#pragma unroll
        for (int j = 0; j < c; ++j) {
          s_mn[j][threadIdx.x] = s_any[threadIdx.x] ? nan_min(s_mn[j][threadIdx.x], s_mn[j][o]) : s_mn[j][o];
          s_mx[j][threadIdx.x] = s_any[threadIdx.x] ? nan_max(s_mx[j][threadIdx.x], s_mx[j][o]) : s_mx[j][o];
        }
        s_any[threadIdx.x] = 1;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    for (int j = 0; j < c; ++j) {
      part[(int64_t)blockIdx.x * 2 * c + j] = s_mn[j][0];
      part[(int64_t)blockIdx.x * 2 * c + c + j] = s_mx[j][0];
    }
  }
}

template <typename T>
static void launch_minmax(const void *x, const int64_t *rows, int64_t n, int c, double *part, int nb, cudaStream_t st) {
  const T *xt = (const T *)x;
  switch (c) {
    case 1: k_aug_minmax_partial<T, 1><<<nb, 256, 0, st>>>(xt, rows, n, part); break;
    case 2: k_aug_minmax_partial<T, 2><<<nb, 256, 0, st>>>(xt, rows, n, part); break;
    case 3: k_aug_minmax_partial<T, 3><<<nb, 256, 0, st>>>(xt, rows, n, part); break;
    default: k_aug_minmax_partial<T, 4><<<nb, 256, 0, st>>>(xt, rows, n, part); break;
  }
}

// one thread per column and side: fold the per-block partials in block order (every block saw at least one row)
__global__ void k_aug_minmax_final(const double *__restrict__ part, int nblocks, int c, double *__restrict__ out) {
  const int t = threadIdx.x;
  if (t >= 2 * c) return;
  double v = part[t];
  for (int b = 1; b < nblocks; ++b) {
    const double w = part[(int64_t)b * 2 * c + t];
    v = t < c ? nan_min(v, w) : nan_max(v, w);
  }
  out[t] = v;
}

// One axis of ndimage.convolve with the (3,) box of float32(1/3): each output is accumulated in double from 0.0 over the
// taps at offsets -1, 0, +1 (out-of-range taps read the constant 0), then rounded once to float32.
__global__ void k_aug_blur_axis(const float *__restrict__ in, float *__restrict__ out, int64_t total, int64_t stride,
                                int64_t dim) {
  const double w = (double)(1.0f / 3.0f);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = (e / stride) % dim;
    const double xm = k > 0 ? (double)in[e - stride] : 0.0;
    const double xp = k < dim - 1 ? (double)in[e + stride] : 0.0;
    double acc = 0.0;
    acc = __dadd_rn(acc, __dmul_rn(xm, w));
    acc = __dadd_rn(acc, __dmul_rn((double)in[e], w));
    acc = __dadd_rn(acc, __dmul_rn(xp, w));
    out[e] = __double2float_rn(acc);
  }
}

// scipy's find_interval_ascending(x, nx, xval, prev_interval=0, extrapolate=1)
__device__ __forceinline__ int find_interval(const double *__restrict__ x, int nx, double xv) {
  const double a = x[0], b = x[nx - 1];
  if (!(a <= xv && xv <= b)) {
    if (xv < a) return 0;
    if (xv > b) return nx - 2;
    return -1;                                             // NaN
  }
  if (xv == b) return nx - 2;
  int low = 0, high = nx - 2;                              // xv >= x[0] = x[prev_interval]
  if (xv < x[low + 1]) high = low;
  while (low < high) {
    const int mid = (high + low) >> 1;
    if (xv < x[mid]) high = mid;
    else if (xv >= x[mid + 1]) low = mid + 1;
    else { low = mid; break; }
  }
  return low;
}

// RegularGridInterpolator 'linear' (scipy 1.18 _rgi.py: find_indices + _evaluate_linear), then p + v * magnitude.
template <typename T>
__global__ void k_aug_elastic_interp(const T *__restrict__ pts, int64_t n, const float *__restrict__ noise, int X, int Y,
                                     int Z, const double *__restrict__ axes, double magnitude, double *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int dims[3] = {X, Y, Z};
  const double *g[3] = {axes, axes + X, axes + X + Y};
  double p[3], y[3];
  int idx[3];
  bool oob = false, nan = false;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    p[d] = (double)pts[3 * i + d];
    nan |= p[d] != p[d];
    oob |= p[d] < g[d][0] || p[d] > g[d][dims[d] - 1];
    idx[d] = find_interval(g[d], dims[d], p[d]);
    y[d] = __ddiv_rn(__dsub_rn(p[d], g[d][idx[d] < 0 ? 0 : idx[d]]),
                     __dsub_rn(g[d][idx[d] + 1], g[d][idx[d] < 0 ? 0 : idx[d]]));
  }
  double v[3] = {0.0, 0.0, 0.0};
  if (nan) {
    v[0] = v[1] = v[2] = __longlong_as_double(0x7ff8000000000000ll);
  } else if (!oob) {
    // the 8 corners in itertools.product order: bit (2 - d) of c selects i + 1 (weight y) over i (weight 1 - y)
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      double wt = 1.0;
      int64_t off = 0;
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const int hi = (c >> (2 - d)) & 1;
        wt = __dmul_rn(wt, hi ? y[d] : __dsub_rn(1.0, y[d]));
        off = off * dims[d] + idx[d] + hi;
      }
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) v[ch] = __dadd_rn(v[ch], __dmul_rn((double)noise[3 * off + ch], wt));
    }
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) out[3 * i + d] = __dadd_rn(p[d], __dmul_rn(v[d], magnitude));
}

// x86 NumPy's float64 -> uint8 cast: truncate to int32 (cvttsd2si; NaN, inf and |x| >= 2^31 give 0x80000000), keep the
// low byte
__device__ __forceinline__ uint8_t np_u8(double x) {
  if (!(x > -2147483649.0 && x < 2147483648.0)) return 0;
  return (uint8_t)(int32_t)x;
}

// np.remainder(x, 1.0): fmod, moved into [0, 1) when negative, +0 for an exact zero
__device__ __forceinline__ double np_rem1(double x) {
  double m = fmod(x, 1.0);
  if (m == 0.0) return 0.0;
  return m < 0.0 ? __dadd_rn(m, 1.0) : m;
}

// np.clip(x, lo, hi): NaN passes, -0.0 stays -0.0
__device__ __forceinline__ double np_clip(double x, double lo, double hi) {
  x = x < lo ? lo : x;
  return x > hi ? hi : x;
}

__device__ __forceinline__ float rsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double rsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float rmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double rmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float radd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double radd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float rdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double rdiv(double a, double b) { return __ddiv_rn(a, b); }

struct AugParams { double keep, blend, tr[3], jitter_scale, hue, sat; };

// CT: coordinate type (float, double or int32); FT: colour type (float or double)
template <typename CT, typename FT>
__global__ void k_aug_input(const CT *__restrict__ coords, const FT *__restrict__ feats, const uint8_t *__restrict__ labels,
                            const int64_t *__restrict__ rows, int64_t n, const double *__restrict__ cmax,
                            const double *__restrict__ fmm, const double *__restrict__ jitter, AugParams P, int32_t stages,
                            int32_t batch, CT *__restrict__ coords_out, FT *__restrict__ feats_out,
                            int32_t *__restrict__ item_coords, float *__restrict__ item_feats,
                            int64_t *__restrict__ item_labels) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const int64_t r = rows ? rows[v] : v;
  // RandomHorizontalFlip: axes 0 then 1, c = max - c in the coordinates' own type
  CT c[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    c[d] = coords[3 * v + d];
    if (d < 2 && (stages & (OSB_AUG_FLIP_X << d))) {
      if constexpr (std::is_integral<CT>::value) c[d] = (CT)cmax[d] - c[d];   // int32: exact
      else c[d] = rsub((CT)cmax[d], c[d]);
    }
  }
  FT f[3];
#pragma unroll
  for (int j = 0; j < 3; ++j) f[j] = feats[3 * r + j];
  if (stages & OSB_AUG_AUTOCONTRAST) {
    // scale = 255 / (hi - lo); f = (1 - b) * f + b * ((f - lo) * scale), all in FT (NumPy keeps float32 for float32)
    const FT keep = (FT)P.keep, blend = (FT)P.blend;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const FT lo = (FT)fmm[j], hi = (FT)fmm[3 + j];
      const FT scale = rdiv((FT)255, rsub(hi, lo));
      const FT cf = rmul(rsub(f[j], lo), scale);
      f[j] = radd(rmul(keep, f[j]), rmul(blend, cf));
    }
  }
  if (stages & OSB_AUG_TRANSLATE) {        // float64 tr + f, clipped, stored back in FT
#pragma unroll
    for (int j = 0; j < 3; ++j) f[j] = (FT)np_clip(__dadd_rn(P.tr[j], (double)f[j]), 0.0, 255.0);
  }
  if (stages & OSB_AUG_JITTER) {           // (randn * (std * 255)) + f, clipped, stored back in FT
#pragma unroll
    for (int j = 0; j < 3; ++j)
      f[j] = (FT)np_clip(__dadd_rn(__dmul_rn(jitter[3 * v + j], P.jitter_scale), (double)f[j]), 0.0, 255.0);
  }
  if (stages & OSB_AUG_HUE_SAT) {
    const double R = (double)f[0], G = (double)f[1], B = (double)f[2];
    // rgb_to_hsv (colorsys order), float64
    const bool anynan = R != R || G != G || B != B;
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    const double maxc = anynan ? qnan : fmax(fmax(R, G), B);
    const double minc = anynan ? qnan : fmin(fmin(R, G), B);
    const bool mask = maxc != minc;
    double s = 0.0, rc = 0.0, gc = 0.0, bc = 0.0;
    if (mask) {
      const double span = __dsub_rn(maxc, minc);
      s = __ddiv_rn(span, maxc);
      rc = __ddiv_rn(__dsub_rn(maxc, R), span);
      gc = __ddiv_rn(__dsub_rn(maxc, G), span);
      bc = __ddiv_rn(__dsub_rn(maxc, B), span);
    }
    double h = R == maxc ? __dsub_rn(bc, gc)
             : G == maxc ? __dsub_rn(__dadd_rn(2.0, rc), bc)
                         : __dsub_rn(__dadd_rn(4.0, gc), rc);
    h = np_rem1(__ddiv_rn(h, 6.0));
    // the translation: h = remainder(hue + h + 1, 1), s = clip(sat * s, 0, 1)
    h = np_rem1(__dadd_rn(__dadd_rn(P.hue, h), 1.0));
    s = np_clip(__dmul_rn(P.sat, s), 0.0, 1.0);
    // hsv_to_rgb: np.select precedence s == 0, i == 1..5, default
    const double h6 = __dmul_rn(h, 6.0);
    const uint8_t i8 = np_u8(h6);
    const double fr = __dsub_rn(h6, (double)i8);
    const double p = __dmul_rn(maxc, __dsub_rn(1.0, s));
    const double q = __dmul_rn(maxc, __dsub_rn(1.0, __dmul_rn(s, fr)));
    const double t = __dmul_rn(maxc, __dsub_rn(1.0, __dmul_rn(s, __dsub_rn(1.0, fr))));
    const int i = i8 % 6;
    double o0, o1, o2;
    if (s == 0.0)    { o0 = maxc; o1 = maxc; o2 = maxc; }
    else if (i == 1) { o0 = q; o1 = maxc; o2 = p; }
    else if (i == 2) { o0 = p; o1 = maxc; o2 = t; }
    else if (i == 3) { o0 = p; o1 = q; o2 = maxc; }
    else if (i == 4) { o0 = t; o1 = p; o2 = maxc; }
    else if (i == 5) { o0 = maxc; o1 = p; o2 = q; }
    else             { o0 = maxc; o1 = t; o2 = p; }
    f[0] = (FT)np_u8(o0);
    f[1] = (FT)np_u8(o1);
    f[2] = (FT)np_u8(o2);
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    if (coords_out) coords_out[3 * v + d] = c[d];
    if (feats_out) feats_out[3 * v + d] = f[d];
  }
  if (item_coords) {                       // [batch, x, y, z] int32 (torch .int() truncates)
    item_coords[4 * v] = batch;
#pragma unroll
    for (int d = 0; d < 3; ++d) item_coords[4 * v + 1 + d] = (int32_t)c[d];
  }
  if (item_feats) {                        // float32(f) / 127.5 - 1 with input_color, else ones
#pragma unroll
    for (int d = 0; d < 3; ++d)
      item_feats[3 * v + d] = (stages & OSB_AUG_INPUT_COLOR) ? __fsub_rn(__fdiv_rn((float)f[d], 127.5f), 1.0f) : 1.0f;
  }
  if (item_labels) item_labels[v] = (int64_t)labels[r];
}

template <typename CT>
static void launch_input(const void *coords, const void *feats, int32_t feats_is_f64, const uint8_t *labels,
                         const int64_t *rows, int64_t n, const double *cmax, const double *fmm, const double *jitter,
                         const AugParams &P, int32_t stages, int32_t batch, void *coords_out, void *feats_out,
                         int32_t *item_coords, float *item_feats, int64_t *item_labels, cudaStream_t stream) {
  const unsigned nb = (unsigned)ceil_div(n, 256);
  if (feats_is_f64)
    k_aug_input<CT, double><<<nb, 256, 0, stream>>>((const CT *)coords, (const double *)feats, labels, rows, n, cmax, fmm,
                                                    jitter, P, stages, batch, (CT *)coords_out, (double *)feats_out,
                                                    item_coords, item_feats, item_labels);
  else
    k_aug_input<CT, float><<<nb, 256, 0, stream>>>((const CT *)coords, (const float *)feats, labels, rows, n, cmax, fmm,
                                                   jitter, P, stages, batch, (CT *)coords_out, (float *)feats_out,
                                                   item_coords, item_feats, item_labels);
}

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_aug_minmax_workspace_bytes(int32_t c) {
  if (c < 1 || c > kMinmaxMaxCols) return 0;
  return (size_t)kMinmaxBlocks * 2 * c * sizeof(double);
}

int osb_aug_minmax(const void *x, int32_t dtype, const int64_t *rows, int64_t n, int32_t c, double *minmax, void *ws,
                   size_t ws_bytes, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n > 0, "osb_aug_minmax: n=%lld must be positive", (long long)n);
  OSB_CHECK(c >= 1 && c <= kMinmaxMaxCols, "osb_aug_minmax: c=%d outside 1..%d", c, kMinmaxMaxCols);
  OSB_CHECK(dtype == AUG_F32 || dtype == AUG_F64 || dtype == AUG_I32, "osb_aug_minmax: dtype code %d (0 f32, 1 f64, 2 i32)",
            dtype);
  OSB_CHECK(x && minmax && ws, "osb_aug_minmax: NULL buffer (x %p, minmax %p, ws %p)", x, (void *)minmax, ws);
  OSB_CHECK(ws_bytes >= osb_aug_minmax_workspace_bytes(c), "osb_aug_minmax: workspace too small (%zu bytes)", ws_bytes);
  const int nb = (int)std::min<int64_t>(kMinmaxBlocks, ceil_div(n, 256));
  double *part = (double *)ws;
  if (dtype == AUG_F32)      launch_minmax<float>(x, rows, n, c, part, nb, stream);
  else if (dtype == AUG_F64) launch_minmax<double>(x, rows, n, c, part, nb, stream);
  else                       launch_minmax<int32_t>(x, rows, n, c, part, nb, stream);
  OSB_LAUNCH_CHECK();
  k_aug_minmax_final<<<1, 32, 0, stream>>>(part, nb, c, minmax);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_aug_blur(float *grid, float *tmp, int32_t X, int32_t Y, int32_t Z, int32_t ch, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(X > 0 && Y > 0 && Z > 0 && ch > 0, "osb_aug_blur: grid %d x %d x %d x %d must be positive", X, Y, Z, ch);
  OSB_CHECK(grid && tmp, "osb_aug_blur: NULL buffer (grid %p, tmp %p)", (void *)grid, (void *)tmp);
  const int64_t total = (int64_t)X * Y * Z * ch;
  OSB_CHECK(total < (1ll << 40), "osb_aug_blur: grid of %lld values too large", (long long)total);
  const int64_t strides[3] = {(int64_t)Y * Z * ch, (int64_t)Z * ch, (int64_t)ch};
  const int64_t dims[3] = {X, Y, Z};
  const unsigned nb = (unsigned)std::min<int64_t>(ceil_div(total, 256), 65536);
  float *src = grid, *dst = tmp;
  for (int pass = 0; pass < 2; ++pass)
    for (int a = 0; a < 3; ++a) {                          // six passes: the result lands back in `grid`
      k_aug_blur_axis<<<nb, 256, 0, stream>>>(src, dst, total, strides[a], dims[a]);
      OSB_LAUNCH_CHECK();
      float *t = src; src = dst; dst = t;
    }
  return 0;
}

int osb_aug_elastic_interp(const void *pts, int32_t pts_is_f64, int64_t n, const float *noise, int32_t X, int32_t Y,
                           int32_t Z, const double *axes, double magnitude, double *out, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n > 0 && n < (1ll << 40), "osb_aug_elastic_interp: n=%lld out of range", (long long)n);
  OSB_CHECK(X >= 2 && Y >= 2 && Z >= 2, "osb_aug_elastic_interp: grid %d x %d x %d needs >= 2 nodes per axis", X, Y, Z);
  OSB_CHECK(pts_is_f64 == 0 || pts_is_f64 == 1, "osb_aug_elastic_interp: pts_is_f64=%d", pts_is_f64);
  OSB_CHECK(pts && noise && axes && out, "osb_aug_elastic_interp: NULL buffer (pts %p, noise %p, axes %p, out %p)", pts,
            (const void *)noise, (const void *)axes, (void *)out);
  const unsigned nb = (unsigned)ceil_div(n, 256);
  if (pts_is_f64)
    k_aug_elastic_interp<double><<<nb, 256, 0, stream>>>((const double *)pts, n, noise, X, Y, Z, axes, magnitude, out);
  else
    k_aug_elastic_interp<float><<<nb, 256, 0, stream>>>((const float *)pts, n, noise, X, Y, Z, axes, magnitude, out);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_aug_input_transforms(const void *coords, int32_t coords_dtype, const void *feats, int32_t feats_is_f64,
                             const uint8_t *labels, const int64_t *rows, int64_t n, const double *coords_max,
                             const double *feats_minmax, const double *jitter, const double *params_host, int32_t stages,
                             int32_t batch_index, void *coords_out, void *feats_out, int32_t *item_coords,
                             float *item_feats, int64_t *item_labels, void *stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  OSB_CHECK(n > 0 && n < (1ll << 40), "osb_aug_input_transforms: n=%lld out of range", (long long)n);
  OSB_CHECK(coords_dtype == AUG_F32 || coords_dtype == AUG_F64 || coords_dtype == AUG_I32,
            "osb_aug_input_transforms: coords dtype code %d (0 f32, 1 f64, 2 i32)", coords_dtype);
  OSB_CHECK(feats_is_f64 == 0 || feats_is_f64 == 1, "osb_aug_input_transforms: feats_is_f64=%d", feats_is_f64);
  OSB_CHECK((stages & ~OSB_AUG_ALL) == 0, "osb_aug_input_transforms: unknown stage bits 0x%x", stages);
  OSB_CHECK(coords && feats && params_host, "osb_aug_input_transforms: NULL buffer (coords %p, feats %p, params %p)",
            coords, feats, (const void *)params_host);
  OSB_CHECK(!(stages & (OSB_AUG_FLIP_X | OSB_AUG_FLIP_Y)) || coords_max,
            "osb_aug_input_transforms: a flip needs the coordinate maxima (NULL buffer)");
  OSB_CHECK(!(stages & OSB_AUG_AUTOCONTRAST) || feats_minmax,
            "osb_aug_input_transforms: auto-contrast needs the colour min / max (NULL buffer)");
  OSB_CHECK(!(stages & OSB_AUG_JITTER) || jitter, "osb_aug_input_transforms: jitter needs its noise (NULL buffer)");
  OSB_CHECK(coords_out || feats_out || item_coords || item_feats || item_labels,
            "osb_aug_input_transforms: no output buffer (all NULL)");
  OSB_CHECK(!item_labels || labels, "osb_aug_input_transforms: item labels need the input labels (NULL buffer)");
  AugParams P;
  P.keep = params_host[0];
  P.blend = params_host[1];
  for (int j = 0; j < 3; ++j) P.tr[j] = params_host[2 + j];
  P.jitter_scale = params_host[5];
  P.hue = params_host[6];
  P.sat = params_host[7];
  if (coords_dtype == AUG_F32)
    launch_input<float>(coords, feats, feats_is_f64, labels, rows, n, coords_max, feats_minmax, jitter, P, stages,
                        batch_index, coords_out, feats_out, item_coords, item_feats, item_labels, stream);
  else if (coords_dtype == AUG_F64)
    launch_input<double>(coords, feats, feats_is_f64, labels, rows, n, coords_max, feats_minmax, jitter, P, stages,
                         batch_index, coords_out, feats_out, item_coords, item_feats, item_labels, stream);
  else
    launch_input<int32_t>(coords, feats, feats_is_f64, labels, rows, n, coords_max, feats_minmax, jitter, P, stages,
                          batch_index, coords_out, feats_out, item_coords, item_feats, item_labels, stream);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
