// TCN / DS-TCN training (tcn_train.cu): the batch-statistics forward with device Dropout masks, and the backward to
// every parameter of the reference's TCN / DS-TCN model with the per-frame linear classifier.  Activations are
// channel-last (M = B * T rows, C channels).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dither.cuh"

namespace wekws {

constexpr int TCN_TRAIN_MAX_LAYERS = 8;
constexpr int TCN_TRAIN_MAX_K = 8;
constexpr int TCN_TRAIN_MAX_IDIM = 128;
constexpr int TCN_TRAIN_MAX_ODIM = 4096;

// The model's dimensions.  Parameters in named_parameters order:
//   0 preprocessing.out.0.weight (C, idim), 1 .bias
//   per block l, from 2 + P l (P = 4 dense, 8 depthwise-separable), backbone.network.l.cnn.:
//     dense: +0 0.weight (C, C, K), +1 0.bias, +2 1.weight, +3 1.bias (BatchNorm)
//     ds:    +0 0.weight (C, 1, K), +1 0.bias, +2 1.weight, +3 1.bias, +4 3.weight (C, C, 1), +5 3.bias, +6 4.weight,
//            +7 4.bias
//   2 + P L classifier.linear.weight (O, C), 3 + P L .bias
// Block l has dilation 2^l and its out_cache columns start at (K - 1)(2^l - 1).
struct TcnTrainDims {
  int C, idim, odim, K, L, ds, act, norm_var;
  int pad_total;
};

// The Dropout of one call: keep element (b, t, c) of block l iff (word >> 8) >= theta[l], word = component c % 4 of
// Philox4x32-10(counter = (c / 4, t, b, 1 + l), key = (seed lo, seed hi)); a kept element is scaled by scale[l].
struct TcnDropout {
  uint64_t seed;
  uint32_t theta[TCN_TRAIN_MAX_LAYERS];
  float scale[TCN_TRAIN_MAX_LAYERS];
};

__host__ __device__ __forceinline__ bool dropout_keep(uint64_t seed, int layer, int b, int t, int c, uint32_t theta) {
  const uint4 w = dither::philox4x32_10(make_uint4((uint32_t)c >> 2, (uint32_t)t, (uint32_t)b, 1u + (uint32_t)layer),
                                        (uint32_t)seed, (uint32_t)(seed >> 32));
  const uint32_t word = (c & 3) == 0 ? w.x : (c & 3) == 1 ? w.y : (c & 3) == 2 ? w.z : w.w;
  return (word >> 8) >= theta;
}

inline int tcn_train_params_per_block(int ds) { return ds ? 8 : 4; }
inline int tcn_train_num_params(const TcnTrainDims& d) { return 4 + tcn_train_params_per_block(d.ds) * d.L; }
inline int tcn_train_num_bns(const TcnTrainDims& d) { return (d.ds ? 2 : 1) * d.L; }
inline int tcn_train_forward_launches(const TcnTrainDims& d) { return 2 + (d.ds ? 2 : 1) * d.L; }
inline int tcn_train_backward_launches(const TcnTrainDims& d) { return 4 + (d.ds ? 3 : 2) * d.L; }

long long tcn_train_saved_floats(const TcnTrainDims& d, long long M);
long long tcn_train_workspace_bytes(const TcnTrainDims& d, long long M, bool save);
long long tcn_backward_workspace_bytes(const TcnTrainDims& d, long long M);

// running: 2 per BatchNorm (running_mean, running_var) in block order (cnn.1[, cnn.4]); bn: (momentum, eps) per
// BatchNorm.  saved == nullptr: nothing is kept for a backward.
int tcn_train_forward_launch(const TcnTrainDims& d, const TcnDropout& drop, const float* feats,
                             const float* const* params, const float* cmvn_mean, const float* cmvn_istd,
                             float* const* running, const double* bn, float* out, float* out_cache, float* saved,
                             void* workspace, int B, int T, cudaStream_t st);
// out: the forward's logits (read when the activation is the sigmoid)
int tcn_backward_launch(const TcnTrainDims& d, const TcnDropout& drop, const float* feats, const float* const* params,
                        const float* cmvn_mean, const float* cmvn_istd, const float* saved, const float* out,
                        const float* grad_out, int B, int T, float* const* grads, void* workspace, cudaStream_t st);
int dropout_mask_launch(uint64_t seed, long long B, long long T, int C, int layer, uint32_t theta, uint8_t* out,
                        cudaStream_t st);

}  // namespace wekws
