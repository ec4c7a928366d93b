// The training step's optimiser on the device: torch.nn.utils.clip_grad_norm_ (L2) and torch.optim.Adam's
// _multi_tensor_adam (L2 weight decay, no amsgrad / maximize / capturable) over a table of tensors passed by value
// in the kernel parameters (up to 32 KB on sm_90 with CUDA >= 12.1), so a step uploads nothing and allocates nothing.
//   * grad_sq_sum_kernel: CTA c of G sums the squares of elements [c E / G, (c + 1) E / G) of the table's
//     concatenated gradients in double (the square of a float32 is exact in double) and writes one partial.
//   * grad_clip_scale_kernel: every CTA adds all partials in the same fixed order (so every CTA forms the same
//     norm), forms torch's clip coefficient and scales its own share of the gradients.  No atomics: equal inputs give
//     equal bits.
//   * adam_kernel: one elementwise pass over 2048-element tiles of the concatenated tensors, with each foreach
//     kernel's float32 rounding of torch's step reproduced in registers (see include/wekws_b200.h).
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace wekws {
namespace {

constexpr int kClipMaxTensors = 1024;   // 16 KB of table per clip launch
constexpr int kAdamMaxTensors = 512;    // 24 KB of table per Adam launch
constexpr int kClipThreads = 256;
constexpr int kClipMaxCtas = 264;       // two per SM on a 132-SM H100; fixed, so the partition is machine-independent
constexpr long long kClipElemsPerCta = 2048;
constexpr int kAdamThreads = 256;
constexpr long long kAdamTile = 2048;

struct ClipTable {
  float* grad[kClipMaxTensors];
  long long start[kClipMaxTensors + 1];  // start[e]: first concatenated index of tensor e; start[n]: the total
  int n;
};

struct AdamTable {
  float* param[kAdamMaxTensors];
  const float* grad[kAdamMaxTensors];
  float* exp_avg[kAdamMaxTensors];
  float* exp_avg_sq[kAdamMaxTensors];
  long long start[kAdamMaxTensors + 1];
  float step_size[kAdamMaxTensors];
  float bc2_sqrt[kAdamMaxTensors];
  int n;
};
static_assert(sizeof(ClipTable) + 64 <= 32764 && sizeof(AdamTable) + 64 <= 32764, "kernel parameter space");

// the last tensor e with start[e] <= i (i < start[n])
__device__ __forceinline__ int find_tensor(const long long* start, int n, long long i) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (start[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// f(e, a, b) for every tensor e overlapping [lo, hi) of the concatenation, a..b the tensor's own element range
template <typename F>
__device__ __forceinline__ void for_each_tensor(const long long* start, int n, long long lo, long long hi, F f) {
  if (lo >= hi) return;
  for (int e = find_tensor(start, n, lo); e < n && start[e] < hi; ++e) {
    const long long a = (lo > start[e] ? lo : start[e]) - start[e];
    const long long b = (hi < start[e + 1] ? hi : start[e + 1]) - start[e];
    if (a < b) f(e, a, b);
  }
}

// the CTA's sum of one double per thread, in a fixed order (warp shuffles, then the warps in order); all threads get it
__device__ __forceinline__ double block_sum(double s) {
  __shared__ double warp_sums[kClipThreads / 32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) warp_sums[threadIdx.x >> 5] = s;
  __syncthreads();
  double t = warp_sums[0];
  for (int w = 1; w < kClipThreads / 32; ++w) t += warp_sums[w];
  return t;
}

__global__ void __launch_bounds__(kClipThreads) grad_sq_sum_kernel(const __grid_constant__ ClipTable t,
                                                                   double* __restrict__ partial) {
  const long long total = t.start[t.n], G = gridDim.x, c = blockIdx.x;
  double s = 0.0;
  for_each_tensor(t.start, t.n, total * c / G, total * (c + 1) / G, [&](int e, long long a, long long b) {
    const float* __restrict__ g = t.grad[e];
    for (long long i = a + threadIdx.x; i < b; i += kClipThreads) {
      const double x = g[i];
      s = fma(x, x, s);
    }
  });
  s = block_sum(s);
  if (threadIdx.x == 0) partial[c] = s;
}

__global__ void __launch_bounds__(kClipThreads) grad_clip_scale_kernel(const __grid_constant__ ClipTable t,
                                                                       const double* __restrict__ partial, int parts,
                                                                       float max_norm, int scale,
                                                                       float* __restrict__ total_norm) {
  double s = 0.0;
  for (int k = threadIdx.x; k < parts; k += kClipThreads) s += partial[k];
  s = block_sum(s);
  const float norm = (float)sqrt(s);
  if (total_norm && blockIdx.x == 0 && threadIdx.x == 0) *total_norm = norm;
  if (!scale) return;
  // torch: clamp(max_norm / (norm + 1e-6), max=1), the division being Tensor.__rdiv__ = reciprocal() * max_norm;
  // the comparison keeps a NaN coefficient NaN, as clamp does
  float coef = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), max_norm);
  coef = coef > 1.0f ? 1.0f : coef;
  const long long total = t.start[t.n], G = gridDim.x, c = blockIdx.x;
  for_each_tensor(t.start, t.n, total * c / G, total * (c + 1) / G, [&](int e, long long a, long long b) {
    float* __restrict__ g = t.grad[e];
    for (long long i = a + threadIdx.x; i < b; i += kClipThreads) g[i] = __fmul_rn(g[i], coef);
  });
}

// torch 2.11 _multi_tensor_adam, one foreach op per line, each rounding to float32 where its kernel stores; an FMA
// where a foreach kernel's `a + s * x` contracts into one, an explicit rounded operation everywhere else
__global__ void __launch_bounds__(kAdamThreads) adam_kernel(const __grid_constant__ AdamTable t, float lerp_w,
                                                            float beta2, float one_minus_beta2, float eps,
                                                            float weight_decay, int use_weight_decay) {
  const long long total = t.start[t.n], lo = blockIdx.x * kAdamTile;
  const long long hi = lo + kAdamTile < total ? lo + kAdamTile : total;
  const bool small_w = fabsf(lerp_w) < 0.5f;
  const float one_minus_w = __fsub_rn(1.0f, lerp_w);
  for_each_tensor(t.start, t.n, lo, hi, [&](int e, long long a, long long b) {
    float* __restrict__ P = t.param[e];
    const float* __restrict__ Gr = t.grad[e];
    float* __restrict__ M = t.exp_avg[e];
    float* __restrict__ V = t.exp_avg_sq[e];
    const float step_size = t.step_size[e], bc2_sqrt = t.bc2_sqrt[e];
    for (long long i = a + threadIdx.x; i < b; i += kAdamThreads) {
      const float p = P[i];
      float g = Gr[i], m = M[i], v = V[i];
      if (use_weight_decay) g = fmaf(weight_decay, p, g);                 // _foreach_add(grads, params, alpha=wd)
      const float d = __fsub_rn(g, m);                                   // _foreach_lerp_(exp_avgs, grads, 1 - beta1)
      m = small_w ? fmaf(lerp_w, d, m) : fmaf(-d, one_minus_w, g);
      v = fmaf(one_minus_beta2, __fmul_rn(g, g), __fmul_rn(v, beta2));  // _foreach_mul_, _foreach_addcmul_
      const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), bc2_sqrt), eps);  // _foreach_sqrt, _div_, _add_
      P[i] = fmaf(step_size, __fdiv_rn(m, denom), p);                     // _foreach_addcdiv_(params, m, denom, ss)
      M[i] = m;
      V[i] = v;
    }
  });
}

int clip_chunks(int n) { return (n + kClipMaxTensors - 1) / kClipMaxTensors; }

int clip_ctas(int64_t total_elems) {
  const int64_t c = (total_elems + kClipElemsPerCta - 1) / kClipElemsPerCta;
  return (int)(c < 1 ? 1 : (c > kClipMaxCtas ? kClipMaxCtas : c));
}

}  // namespace
}  // namespace wekws

using namespace wekws;

extern "C" int64_t wekws_grad_clip_workspace_bytes(int n, int64_t total_elems) {
  if (n < 0 || total_elems < 0) return WEKWS_ERR_INVALID;
  if (n == 0 || total_elems == 0) return 0;
  return (int64_t)sizeof(double) * clip_chunks(n) * clip_ctas(total_elems);
}

extern "C" int wekws_grad_clip_launches(int n) { return n > 0 ? 2 * clip_chunks(n) : 0; }

extern "C" int wekws_adam_step_launches(int n) {
  return n > 0 ? (n + kAdamMaxTensors - 1) / kAdamMaxTensors : 0;
}

extern "C" int wekws_grad_clip(float* const* h_grads, const int64_t* h_numel, int n, double max_norm,
                               float* d_total_norm, void* d_workspace, void* stream) {
  WEKWS_REQUIRE(n >= 0, "wekws_grad_clip: bad tensor count %d", n);
  if (n == 0) return WEKWS_OK;
  WEKWS_REQUIRE(h_grads && h_numel && d_total_norm && d_workspace, "wekws_grad_clip: null argument");
  int64_t total = 0;
  for (int i = 0; i < n; ++i) {
    WEKWS_REQUIRE(h_grads[i] && h_numel[i] >= 1, "wekws_grad_clip: tensor %d is null or empty (numel %lld)", i,
                  (long long)h_numel[i]);
    total += h_numel[i];
  }
  const int G = clip_ctas(total), chunks = clip_chunks(n);
  const bool scale = !isnan(max_norm);
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = static_cast<double*>(d_workspace);
  ClipTable t;
  for (int pass = 0; pass < 2; ++pass)
    for (int k = 0; k < chunks; ++k) {
      const int i0 = k * kClipMaxTensors, cnt = n - i0 < kClipMaxTensors ? n - i0 : kClipMaxTensors;
      t.n = cnt;
      t.start[0] = 0;
      for (int e = 0; e < cnt; ++e) {
        t.grad[e] = h_grads[i0 + e];
        t.start[e + 1] = t.start[e] + h_numel[i0 + e];
      }
      int rc;
      if (pass == 0) {
        grad_sq_sum_kernel<<<G, kClipThreads, 0, st>>>(t, partial + (int64_t)k * G);
        rc = check_launch("grad_sq_sum_kernel");
      } else {
        grad_clip_scale_kernel<<<G, kClipThreads, 0, st>>>(t, partial, chunks * G, (float)max_norm, scale ? 1 : 0,
                                                           k == 0 ? d_total_norm : nullptr);
        rc = check_launch("grad_clip_scale_kernel");
      }
      if (rc != WEKWS_OK) return rc;
    }
  return WEKWS_OK;
}

extern "C" int wekws_adam_step(float* const* h_params, const float* const* h_grads, float* const* h_exp_avg,
                               float* const* h_exp_avg_sq, const int64_t* h_numel, const double* h_step_size,
                               const double* h_bc2_sqrt, int n, double beta1, double beta2, double eps,
                               double weight_decay, void* stream) {
  WEKWS_REQUIRE(n >= 0, "wekws_adam_step: bad tensor count %d", n);
  if (n == 0) return WEKWS_OK;
  WEKWS_REQUIRE(h_params && h_grads && h_exp_avg && h_exp_avg_sq && h_numel && h_step_size && h_bc2_sqrt,
                "wekws_adam_step: null argument");
  for (int i = 0; i < n; ++i)
    WEKWS_REQUIRE(h_params[i] && h_grads[i] && h_exp_avg[i] && h_exp_avg_sq[i] && h_numel[i] >= 1,
                  "wekws_adam_step: tensor %d is null or empty (numel %lld)", i, (long long)h_numel[i]);
  cudaStream_t st = (cudaStream_t)stream;
  AdamTable t;
  for (int i0 = 0; i0 < n; i0 += kAdamMaxTensors) {
    const int cnt = n - i0 < kAdamMaxTensors ? n - i0 : kAdamMaxTensors;
    t.n = cnt;
    t.start[0] = 0;
    for (int e = 0; e < cnt; ++e) {
      t.param[e] = h_params[i0 + e];
      t.grad[e] = h_grads[i0 + e];
      t.exp_avg[e] = h_exp_avg[i0 + e];
      t.exp_avg_sq[e] = h_exp_avg_sq[i0 + e];
      t.start[e + 1] = t.start[e] + h_numel[i0 + e];
      t.step_size[e] = (float)h_step_size[i0 + e];
      t.bc2_sqrt[e] = (float)h_bc2_sqrt[i0 + e];
    }
    const long long tiles = (t.start[cnt] + kAdamTile - 1) / kAdamTile;
    WEKWS_REQUIRE(tiles < (1ll << 31), "wekws_adam_step: %lld elements is more than one launch handles",
                  (long long)t.start[cnt]);
    adam_kernel<<<(unsigned)tiles, kAdamThreads, 0, st>>>(t, (float)(1.0 - beta1), (float)beta2,
                                                          (float)(1.0 - beta2), (float)eps, (float)weight_decay,
                                                          weight_decay != 0.0 ? 1 : 0);
    const int rc = check_launch("adam_kernel");
    if (rc != WEKWS_OK) return rc;
  }
  return WEKWS_OK;
}
