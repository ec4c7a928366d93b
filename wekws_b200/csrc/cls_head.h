// Kernel argument block of the utterance-level classifier heads (cls_head.cu).
#pragma once
#include <cuda_runtime.h>

namespace wekws {

constexpr int kHeadWidth = 64;     // Linear(hidden, 64) -> ReLU -> Linear(64, odim), as the reference hard-codes it

struct ClsHeadArgs {
  const float* pool;       // (B, H) pooled backbone output: sum over the frames the head reads
  float* out;              // (B, odim)
  const float* vec;        // per-channel vector blob; the head's weights live at the offsets below
  int B, H, odim, act, softmax;
  float scale;             // 1 / T for the global head, 1 for the last-frame head
  int v_w0, v_b0, v_w1, v_b1;   // W0^T [H][64], b0 [64], W1^T [64][odim], b1 [odim]
};

int cls_head_launch(const ClsHeadArgs& a, cudaStream_t st);

}  // namespace wekws
