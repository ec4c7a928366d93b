// Shared host/device helpers for the wekws_b200 C-ABI library (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>
#include <string>

#include "../../include/wekws_b200.h"

namespace wekws {

// ---- error plumbing: thread-local message, negative status codes, no exceptions ----
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launches;

#define WEKWS_CUDA_OK(expr)                                                          \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) {                                                         \
      ::wekws::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),     \
                         __FILE__, __LINE__);                                        \
      return WEKWS_ERR_CUDA;                                                         \
    }                                                                                \
  } while (0)

#define WEKWS_REQUIRE(cond, ...)                                                     \
  do {                                                                               \
    if (!(cond)) {                                                                   \
      ::wekws::set_error(__VA_ARGS__);                                               \
      return WEKWS_ERR_INVALID;                                                      \
    }                                                                                \
  } while (0)

inline int check_launch(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("launch of %s failed: %s", what, cudaGetErrorString(e));
    return WEKWS_ERR_CUDA;
  }
  return WEKWS_OK;
}

int device_sm_count();
// Lets `kernel` launch on the current device with `bytes` of dynamic shared memory: raises its limit when needed,
// never lowers it.  Thread-safe.
int opt_in_smem(const void* kernel, size_t bytes);

// ---- device helpers ----
#ifdef __CUDACC__
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) {
  unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
  unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem_dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
// Wait until at most `pending` most-recently committed groups are still in flight.
__device__ __forceinline__ void cp_async_wait_pending(int pending) {
  switch (pending) {
    case 0: asm volatile("cp.async.wait_group 0;\n" ::); break;
    case 1: asm volatile("cp.async.wait_group 1;\n" ::); break;
    case 2: asm volatile("cp.async.wait_group 2;\n" ::); break;
    default: asm volatile("cp.async.wait_group 3;\n" ::); break;
  }
}
__device__ __forceinline__ float sigmoidf_acc(float x) { return 1.0f / (1.0f + expf(-x)); }

// The double Python parses back from '{:.6f}'.format(x) (the score file of wekws/bin/score.py:128-137): x * 1e6 is
// exact in double for a float x in [0, 1] (24 x 20 significant bits), so rint of it is the 6-decimal text value.
// The DET sweep and the online threshold detector compare scores through this one definition.
__device__ __forceinline__ double text_round6(float x) { return rint((double)x * 1e6) / 1e6; }

// Softmax normaliser of the row p[0..n) across one warp: every lane gets m = max p and s = sum expf(p[i] - m), and
// the row's softmax is expf(p[i] - m) / s.  The model's softmax and the CTC criterion (log-softmax, and the
// posteriors its accuracy decodes) share this code, so their probabilities are bit-identical.
__device__ __forceinline__ void warp_row_max_sum(const float* p, int n, int lane, float& m, float& s) {
  m = -INFINITY;
  for (int i = lane; i < n; i += 32) m = fmaxf(m, p[i]);
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  s = 0.f;
  for (int i = lane; i < n; i += 32) s += expf(p[i] - m);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
}
#endif

}  // namespace wekws
