// Optimiser step of the fused training engine on the device, and the in-place re-pack of its tensor-core operands:
//   osb_optim_adam   torch.optim.Adam's foreach update (_multi_tensor_adam, no amsgrad / maximize / weight decay)
//   osb_optim_sgd    torch.optim.SGD's foreach update (_multi_tensor_sgd, no nesterov / dampening)
//   osb_conv_repack  the split-bf16 B operands (osb_conv_pack_weights' layout) of many weights into existing buffers
// Each is one launch over a device table, multi-tensor-apply style: block-sized chunks of one tensor each, float4 accesses
// where every stream of the tensor shares the same 16-byte phase, scalar heads and tails otherwise.
// The build contracts a*b+c into FMAs, so every rounding step of the updates is spelled with an explicit intrinsic, in the
// order torch's CUDA foreach kernels round (DESIGN.md "Optimiser contract").
#include "common.cuh"

#include <algorithm>

namespace osb {

static_assert(sizeof(osb_adam_tensor) == 72, "osb_adam_tensor layout");
static_assert(sizeof(osb_sgd_tensor) == 56, "osb_sgd_tensor layout");
static_assert(sizeof(osb_pack_job) == 64, "osb_pack_job layout");

static constexpr int kOptimThreads = 256;
static constexpr int kMaxBlocks = 132 * 16;

// index of the table entry owning chunk ch: the last j with tab[j].chunk_begin <= ch
template <typename T>
__device__ __forceinline__ int find_entry(const T *__restrict__ tab, int n, int64_t ch) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (tab[mid].chunk_begin <= ch) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// torch's lerp (ATen/native/Lerp.h) as its CUDA build contracts it: self + w (end - self) for |w| < 0.5, else
// end - (end - self)(1 - w)
__device__ __forceinline__ float lerp_torch(float self, float end, float w) {
  const float d = __fsub_rn(end, self);
  return fabsf(w) < 0.5f ? __fmaf_rn(w, d, self) : __fmaf_rn(-d, __fsub_rn(1.f, w), end);
}

__device__ __forceinline__ void adam_elem(float &p, float g, float &m, float &v, const osb_adam_tensor &t) {
  m = lerp_torch(m, g, t.lerp_w);                                              // _foreach_lerp_(m, g, 1 - beta1)
  v = __fmaf_rn(t.one_minus_beta2, __fmul_rn(g, g), __fmul_rn(v, t.beta2));   // _foreach_mul_, _foreach_addcmul_
  const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), t.bc2_sqrt), t.eps); // _foreach_sqrt, _foreach_div_, _foreach_add_
  p = __fmaf_rn(t.step_size, __fdiv_rn(m, denom), p);                          // _foreach_addcdiv_(p, m, denom, step_size)
}

__device__ __forceinline__ void sgd_elem(float &p, float g, float *b, const osb_sgd_tensor &t) {
  float d = t.weight_decay != 0.f ? __fmaf_rn(t.weight_decay, p, g) : g;      // _foreach_add(g, p, alpha=weight_decay)
  if (b) {
    d = t.first ? d : __fadd_rn(__fmul_rn(*b, t.momentum), d);                 // clone, or _foreach_mul_ then _foreach_add_
    *b = d;
  }
  p = __fmaf_rn(t.neg_lr, d, p);                                               // _foreach_add_(p, d, alpha=-lr)
}

__device__ __forceinline__ bool aligned_with(const void *a, uintptr_t phase) {
  return a == nullptr || ((uintptr_t)a & 15) == phase;
}

// [lo, hi) of a chunk split into a scalar head [lo, a0), a float4 body [a0, a1) and a scalar tail [a1, hi)
__device__ __forceinline__ void chunk_split(bool vec, uintptr_t phase, int64_t lo, int64_t hi, int64_t &a0, int64_t &a1) {
  if (!vec) { a0 = a1 = hi; return; }
  a0 = std::min(hi, lo + (int64_t)(((16 - phase) & 15) >> 2));      // lo is a multiple of 4: the head is the tensor's
  a1 = a0 + ((hi - a0) & ~(int64_t)3);
}

__global__ void __launch_bounds__(kOptimThreads) k_optim_adam(const osb_adam_tensor *__restrict__ tab, int n,
                                                               int64_t chunk_elems, int64_t n_chunks) {
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    const osb_adam_tensor t = tab[find_entry(tab, n, ch)];
    const int64_t lo = (ch - t.chunk_begin) * chunk_elems, hi = std::min(lo + chunk_elems, t.numel);
    const uintptr_t phase = (uintptr_t)t.param & 15;
    const bool vec = (phase & 3) == 0 && aligned_with(t.grad, phase) && aligned_with(t.exp_avg, phase) &&
                     aligned_with(t.exp_avg_sq, phase);
    int64_t a0, a1;
    chunk_split(vec, phase, lo, hi, a0, a1);
    for (int64_t e = a0 + 4 * (int64_t)threadIdx.x; e < a1; e += 4 * (int64_t)blockDim.x) {
      float4 p = *reinterpret_cast<const float4 *>(t.param + e);
      const float4 g = *reinterpret_cast<const float4 *>(t.grad + e);
      float4 m = *reinterpret_cast<const float4 *>(t.exp_avg + e);
      float4 v = *reinterpret_cast<const float4 *>(t.exp_avg_sq + e);
      adam_elem(p.x, g.x, m.x, v.x, t);
      adam_elem(p.y, g.y, m.y, v.y, t);
      adam_elem(p.z, g.z, m.z, v.z, t);
      adam_elem(p.w, g.w, m.w, v.w, t);
      *reinterpret_cast<float4 *>(t.param + e) = p;
      *reinterpret_cast<float4 *>(t.exp_avg + e) = m;
      *reinterpret_cast<float4 *>(t.exp_avg_sq + e) = v;
    }
    const int64_t n_head = a0 - lo;
    for (int64_t i = threadIdx.x; i < n_head + (hi - a1); i += blockDim.x) {
      const int64_t e = i < n_head ? lo + i : a1 + (i - n_head);
      float p = t.param[e], m = t.exp_avg[e], v = t.exp_avg_sq[e];
      adam_elem(p, t.grad[e], m, v, t);
      t.param[e] = p;
      t.exp_avg[e] = m;
      t.exp_avg_sq[e] = v;
    }
  }
}

__global__ void __launch_bounds__(kOptimThreads) k_optim_sgd(const osb_sgd_tensor *__restrict__ tab, int n,
                                                              int64_t chunk_elems, int64_t n_chunks) {
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    const osb_sgd_tensor t = tab[find_entry(tab, n, ch)];
    const int64_t lo = (ch - t.chunk_begin) * chunk_elems, hi = std::min(lo + chunk_elems, t.numel);
    const uintptr_t phase = (uintptr_t)t.param & 15;
    const bool vec = (phase & 3) == 0 && aligned_with(t.grad, phase) && aligned_with(t.momentum_buffer, phase);
    int64_t a0, a1;
    chunk_split(vec, phase, lo, hi, a0, a1);
    for (int64_t e = a0 + 4 * (int64_t)threadIdx.x; e < a1; e += 4 * (int64_t)blockDim.x) {
      float4 p = *reinterpret_cast<const float4 *>(t.param + e);
      const float4 g = *reinterpret_cast<const float4 *>(t.grad + e);
      if (t.momentum_buffer) {
        float4 b = t.first ? make_float4(0.f, 0.f, 0.f, 0.f) : *reinterpret_cast<const float4 *>(t.momentum_buffer + e);
        sgd_elem(p.x, g.x, &b.x, t);
        sgd_elem(p.y, g.y, &b.y, t);
        sgd_elem(p.z, g.z, &b.z, t);
        sgd_elem(p.w, g.w, &b.w, t);
        *reinterpret_cast<float4 *>(t.momentum_buffer + e) = b;
      } else {
        sgd_elem(p.x, g.x, nullptr, t);
        sgd_elem(p.y, g.y, nullptr, t);
        sgd_elem(p.z, g.z, nullptr, t);
        sgd_elem(p.w, g.w, nullptr, t);
      }
      *reinterpret_cast<float4 *>(t.param + e) = p;
    }
    const int64_t n_head = a0 - lo;
    for (int64_t i = threadIdx.x; i < n_head + (hi - a1); i += blockDim.x) {
      const int64_t e = i < n_head ? lo + i : a1 + (i - n_head);
      float p = t.param[e];
      if (t.momentum_buffer) {
        float b = t.first ? 0.f : t.momentum_buffer[e];
        sgd_elem(p, t.grad[e], &b, t);
        t.momentum_buffer[e] = b;
      } else {
        sgd_elem(p, t.grad[e], nullptr, t);
      }
      t.param[e] = p;
    }
  }
}

__global__ void __launch_bounds__(kOptimThreads) k_conv_repack(const osb_pack_job *__restrict__ jobs, int n,
                                                                int64_t chunk_elems, int64_t n_chunks) {
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    const osb_pack_job j = jobs[find_entry(jobs, n, ch)];
    const int64_t total = (int64_t)j.K * j.cout_pad * j.cin;
    const int64_t lo = (ch - j.chunk_begin) * chunk_elems, hi = std::min(lo + chunk_elems, total);
    for (int64_t e = lo + threadIdx.x; e < hi; e += blockDim.x)
      pack_weight_elem(j.w, j.sk, j.sn, j.sc, j.cin, j.cout, j.cout_pad, e, (uint8_t *)j.wpack);
  }
}

static int check_table(const char *what, const void *table, int32_t n, int64_t chunk_elems, int64_t n_chunks, int vec4) {
  OSB_CHECK(table != nullptr, "%s: NULL table", what);
  OSB_CHECK(n >= 1, "%s: %d table entries (need >= 1)", what, n);
  OSB_CHECK(chunk_elems >= 1 && (!vec4 || chunk_elems % 4 == 0), "%s: chunk_elems %lld must be positive%s", what,
            (long long)chunk_elems, vec4 ? " and a multiple of 4" : "");
  OSB_CHECK(n_chunks >= n, "%s: %lld chunks for %d entries (every entry owns at least one)", what, (long long)n_chunks, n);
  return 0;
}

static unsigned grid_of(int64_t n_chunks) { return (unsigned)std::min<int64_t>(n_chunks, kMaxBlocks); }

}  // namespace osb

using namespace osb;

extern "C" {

size_t osb_optim_entry_bytes(int32_t kind) {
  switch (kind) {
    case 0: return sizeof(osb_adam_tensor);
    case 1: return sizeof(osb_sgd_tensor);
    case 2: return sizeof(osb_pack_job);
    default: return 0;
  }
}

int osb_optim_adam(const osb_adam_tensor *table, int32_t n_tensors, int64_t chunk_elems, int64_t n_chunks, void *stream) {
  if (check_table("osb_optim_adam", table, n_tensors, chunk_elems, n_chunks, 1)) return 1;
  k_optim_adam<<<grid_of(n_chunks), kOptimThreads, 0, (cudaStream_t)stream>>>(table, n_tensors, chunk_elems, n_chunks);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_optim_sgd(const osb_sgd_tensor *table, int32_t n_tensors, int64_t chunk_elems, int64_t n_chunks, void *stream) {
  if (check_table("osb_optim_sgd", table, n_tensors, chunk_elems, n_chunks, 1)) return 1;
  k_optim_sgd<<<grid_of(n_chunks), kOptimThreads, 0, (cudaStream_t)stream>>>(table, n_tensors, chunk_elems, n_chunks);
  OSB_LAUNCH_CHECK();
  return 0;
}

int osb_conv_repack(const osb_pack_job *jobs, int32_t n_jobs, int64_t chunk_elems, int64_t n_chunks, void *stream) {
  if (check_table("osb_conv_repack", jobs, n_jobs, chunk_elems, n_chunks, 0)) return 1;
  k_conv_repack<<<grid_of(n_chunks), kOptimThreads, 0, (cudaStream_t)stream>>>(jobs, n_jobs, chunk_elems, n_chunks);
  OSB_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
