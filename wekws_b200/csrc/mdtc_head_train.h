// MDTC training with the speech-command heads (mdtc_head_train.cu): the batch-statistics forward of the MDTC backbone
// (mdtc_train.cu, without its classifier) followed by the `global` / `last` head's training forward with a device
// Dropout mask, and the backward to every parameter.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "mdtc_train.h"

namespace wekws {

constexpr int MDTC_HEAD_WIDTH = 64;              // Linear(C, 64) -> ReLU -> Dropout -> Linear(64, odim)
constexpr int MDTC_HEAD_TRAIN_MAX_ODIM = 4096;
constexpr int MDTC_HEAD_DROPOUT_LAYER = 255;     // dropout_keep's layer: Philox counter word 3 = 256

// The head of one call.  Parameters in named_parameters order: the MDTC backbone's 2 + 12 L (mdtc_train.h), then
//   2 + 12 L classifier.classifier.0.weight (64, C), 3 + 12 L .bias, 4 + 12 L classifier.classifier.3.weight
//   (odim, 64), 5 + 12 L .bias.
// Dropout: element (b, j) is kept iff dropout_keep(seed, 255, b, 0, j, theta) (tcn_train.h); kept: times scale.
struct MdtcHead {
  int last;                // 0: mean over all T frames (global), 1: frame T - 1 (last)
  int odim;
  uint64_t seed;
  uint32_t theta;
  float scale;
};

inline int mdtc_head_train_num_params(int L) { return 6 + 12 * L; }
inline int mdtc_head_train_forward_launches(int L) { return 3 + 3 * L; }
inline int mdtc_head_backward_launches(int L) { return 4 + 4 * L; }

// d: the backbone's dimensions with odim = 0
long long mdtc_head_train_saved_floats(const MdtcTrainDims& d, long long B, long long T);
long long mdtc_head_train_workspace_bytes(const MdtcTrainDims& d, long long B, long long T, bool save);
long long mdtc_head_backward_workspace_bytes(const MdtcTrainDims& d, long long B, long long T);

int mdtc_head_train_forward_launch(const MdtcTrainDims& d, const MdtcHead& h, const float* feats,
                                   const float* const* params, const float* cmvn_mean, const float* cmvn_istd,
                                   float* const* running, const double* bn, float* out, float* out_cache, float* saved,
                                   void* workspace, int B, int T, cudaStream_t st);
int mdtc_head_backward_launch(const MdtcTrainDims& d, const MdtcHead& h, const float* feats,
                              const float* const* params, const float* cmvn_mean, const float* cmvn_istd,
                              const float* saved, const float* grad_out, int B, int T, float* const* grads,
                              void* workspace, cudaStream_t st);

}  // namespace wekws
