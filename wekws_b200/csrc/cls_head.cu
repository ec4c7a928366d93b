// Utterance-level classifier heads of the speech-command recipes: GlobalClassifier / LastClassifier around
// Sequential(Linear(hidden, 64), ReLU, Dropout, Linear(64, odim)) (reference wekws/model/classifier.py:19-40,
// kws_model.py:175-195), then the activation and the optional softmax (kws_model.py:78-90).
//
// The backbone kernels leave the per-stream pooled vector (sum over the frames the head reads) in a (B, H) buffer;
// this kernel does the rest, one CTA of 64 threads per stream.  That is 64 H + 64 odim MACs per stream per call, not
// per frame, so it runs in FP32 FMA: tensor cores would buy nothing here.
#include "cls_head.h"
#include "common.cuh"

namespace wekws {

namespace {

constexpr int NT_HEAD = kHeadWidth;      // one thread per hidden unit of the MLP

__global__ void __launch_bounds__(NT_HEAD) cls_head_kernel(const ClsHeadArgs a) {
  extern __shared__ float sm[];
  float* x = sm;                          // [H]
  float* h = x + a.H;                     // [64]
  float* y = h + kHeadWidth;              // [odim]
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* p = a.pool + (size_t)b * a.H;
  for (int c = tid; c < a.H; c += NT_HEAD) x[c] = p[c] * a.scale;     // the mean over T frames (global) or frame T-1
  __syncthreads();
  {
    const float* w0 = a.vec + a.v_w0 + tid;
    float acc = __ldg(a.vec + a.v_b0 + tid);
#pragma unroll 8
    for (int c = 0; c < a.H; ++c) acc = fmaf(__ldg(w0 + c * kHeadWidth), x[c], acc);
    h[tid] = fmaxf(acc, 0.f);            // ReLU; Dropout is the identity in eval mode
  }
  __syncthreads();
  for (int j = tid; j < a.odim; j += NT_HEAD) {
    const float* w1 = a.vec + a.v_w1 + j;
    float acc = __ldg(a.vec + a.v_b1 + j);
#pragma unroll 8
    for (int k = 0; k < kHeadWidth; ++k) acc = fmaf(__ldg(w1 + k * a.odim), h[k], acc);
    if (a.act == WEKWS_ACT_SIGMOID) acc = sigmoidf_acc(acc);
    y[j] = acc;
  }
  float* o = a.out + (size_t)b * a.odim;
  if (!a.softmax) {
    for (int j = tid; j < a.odim; j += NT_HEAD) o[j] = y[j];
    return;
  }
  __syncthreads();
  if (tid >= 32) return;                  // softmax over the row by warp 0, butterflies in a fixed order
  float m = -INFINITY;
  for (int j = tid; j < a.odim; j += 32) m = fmaxf(m, y[j]);
  for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
  float z = 0.f;
  for (int j = tid; j < a.odim; j += 32) z += expf(y[j] - m);
  for (int s = 16; s > 0; s >>= 1) z += __shfl_xor_sync(0xffffffffu, z, s);
  for (int j = tid; j < a.odim; j += 32) o[j] = expf(y[j] - m) / z;
}

}  // namespace

int cls_head_launch(const ClsHeadArgs& a, cudaStream_t st) {
  WEKWS_REQUIRE(a.B >= 1 && a.H >= 1 && a.odim >= 1, "cls_head_launch: bad shape");
  const size_t smem = (size_t)(a.H + kHeadWidth + a.odim) * sizeof(float);
  if (const int rc = opt_in_smem((const void*)cls_head_kernel, smem)) return rc;
  cls_head_kernel<<<(unsigned)a.B, NT_HEAD, smem, st>>>(a);
  return check_launch("cls_head_kernel");
}

}  // namespace wekws
