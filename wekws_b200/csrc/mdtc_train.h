// MDTC training (mdtc_train.cu): the batch-statistics forward and the backward to every parameter of the reference's
// MDTC model with the per-frame linear classifier.  Activations are channel-last (M = B * T rows, C channels).
#pragma once
#include <cuda_runtime.h>

namespace wekws {

constexpr int MDTC_TRAIN_SLICES = 128;      // fixed row slices of every batch statistic and weight-gradient sum
constexpr int MDTC_TRAIN_MAX_BLOCKS = 25;   // preprocessor + stacks
constexpr int MDTC_TRAIN_MAX_K = 8;
constexpr int MDTC_TRAIN_MAX_ODIM = 16;
constexpr int MDTC_TRAIN_MAX_IDIM = 128;

// The model's dimensions and, per call, the device tensors the kernels read.  Parameters in named_parameters order:
//   0 preprocessing.out.0.weight (C, idim), 1 .bias
//   per block b (preprocessor, then the stacks' res_blocks), from 2 + 12 b:
//     +0 conv1.conv.weight (C, 1, K), +1 .bias, +2 conv1.bn.weight, +3 .bias, +4 conv1.pointwise.weight (C, C, 1),
//     +5 .bias, +6 bn1.weight, +7 .bias, +8 conv2.weight (C, C, 1), +9 .bias, +10 bn2.weight, +11 .bias
//   2 + 12 L classifier.linear.weight (O, C), 3 + 12 L .bias
// odim = 0: no classifier (mdtc_head_train.cu).  The forward's output is the stack sum, kept where
// mdtc_train_stack_sum says, and `out` is not written; the backward's grad_out is the stack sum's gradient (B, T, C),
// and the classifier parameters and gradients are neither read nor written.
struct MdtcTrainDims {
  int C, idim, odim, K, L, stack_size, act, norm_var;
  int dil[MDTC_TRAIN_MAX_BLOCKS], coff[MDTC_TRAIN_MAX_BLOCKS];   // per block: dilation, offset in the cache
  int pad_total;
};

inline int mdtc_train_num_params(int L) { return 4 + 12 * L; }
inline int mdtc_train_forward_launches(int L) { return 2 + 3 * L; }
inline int mdtc_train_backward_launches(int L) { return 3 + 4 * L; }
// a stack's last block: its output is a term of the backbone's output sum
inline bool mdtc_stack_end(int b, int stack_size) { return b > 0 && b % stack_size == 0; }

long long mdtc_train_saved_floats(const MdtcTrainDims& d, long long M);
long long mdtc_train_workspace_bytes(const MdtcTrainDims& d, long long M, bool save);
long long mdtc_backward_workspace_bytes(const MdtcTrainDims& d, long long M);
// where the forward leaves the stack sum (B, T, C): in `saved` when it is kept, else in `workspace`
float* mdtc_train_stack_sum(const MdtcTrainDims& d, long long M, float* saved, void* workspace);

// running: 2 per BatchNorm (running_mean, running_var) in block order bn0, bn1, bn2; bn: (momentum, eps) per BatchNorm.
// saved == nullptr: nothing is kept for a backward.
int mdtc_train_forward_launch(const MdtcTrainDims& d, const float* feats, const float* const* params,
                              const float* cmvn_mean, const float* cmvn_istd, float* const* running, const double* bn,
                              float* out, float* out_cache, float* saved, void* workspace, int B, int T,
                              cudaStream_t st);
int mdtc_backward_launch(const MdtcTrainDims& d, const float* feats, const float* const* params,
                         const float* cmvn_mean, const float* cmvn_istd, const float* saved, const float* grad_out,
                         int B, int T, float* const* grads, void* workspace, cudaStream_t st);

}  // namespace wekws
