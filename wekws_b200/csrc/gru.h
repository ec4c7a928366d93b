// Kernel argument block of the fused GRU kernel (gru.cu).
#pragma once
#include <cuda_runtime.h>

namespace wekws {

struct GruArgs {
  const float* feats;      // (B, T, idim)
  const float* in_cache;   // (L, B, H) or nullptr (== zeros)
  float* out;              // (B, T, odim)
  float* out_cache;        // (L, B, H)
  const float* vec;        // packed weights (see model_host.cu: pack_gru)
  int B, T, L, H, idim, odim, act, has_cmvn;
  int v_mean, v_istd, v_wp, v_bp, v_layers, v_layer_stride, v_wc, v_bc;
  int n_tiles;
  // training forward only: the activations the backward reads, (1 + 5 L) consecutive (B * T, H) row-major blocks,
  // row b * T + t: the layer-0 input x0 = ReLU(Linear(CMVN(feats))), then per layer l: h_t, r, z, n and
  // hn = W_hn h_{t-1} + b_hn (gru_saved_block)
  float* saved;
};

// first float of saved block `which` (0 h, 1 r, 2 z, 3 n, 4 hn) of layer l; the layer-0 input is block 0
inline long long gru_saved_block(long long M, int H, int l, int which) { return M * H * (1 + 5LL * l + which); }
inline long long gru_saved_per_frame(int L, int H) { return (1 + 5LL * L) * H; }

// save: the training forward, from empty caches (in_cache == nullptr), also writing a.saved
int gru_launch(const GruArgs& a, cudaStream_t st, bool save = false);

// gru_train.cu -------------------------------------------------------------------------------------------------------
// Parameters in named_parameters order: preprocessing.out.0.{weight,bias}, per layer backbone.{weight_ih, weight_hh,
// bias_ih, bias_hh}_l{k}, classifier.linear.{weight,bias}.
int gru_num_params(int L);                                   // 4 + 4 L
int gru_backward_launches(int L);                            // 5 + 4 L
long long gru_backward_workspace_floats(const GruArgs& a, long long M);
// Backward of a training forward over B utterances of T frames from `saved` and its logits `out`; grads[i] in
// parameter order, every element written.
int gru_backward_launch(const GruArgs& a, const float* feats, const float* saved, const float* out,
                        const float* grad_out, int B, int T, float* const* grads, float* workspace, cudaStream_t st);

}  // namespace wekws
