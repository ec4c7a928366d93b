// Kernel argument block of the fused FSMN kernel (fsmn.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

namespace wekws {

struct FsmnArgs {
  const float* feats;      // (B, T, idim), stream stride feat_bstride
  const float* in_cache;   // (B, proj, pad, L) or nullptr (start of stream == zeros)
  float* out;              // (B, T, odim), stream stride out_bstride
  float* out_cache;        // (B, proj, pad, L); may alias in_cache
  const float* w;          // packed weights (model_host.cu pack_fsmn): transposed, column-padded matrices + vectors
  int B, T, S, n_tiles;
  long long feat_bstride, out_bstride;
  int idim, aff_in, lin, proj, aff_out, odim, L, lorder, rorder, act, has_cmvn, norm_var;
  int np_aff_in, np_lin, np_proj, np_aff_out, np_odim;     // output widths padded to the 128-column GEMM pass
  int sp0, sp1, spm;                                       // row strides (floats) of the shared activation buffers
  int o_mean, o_istd, o_w_in1, o_b_in1, o_w_in2, o_b_in2, o_w_out1, o_b_out1, o_w_out2, o_b_out2;
  int o_layers, layer_stride, lo_wp, lo_taps, lo_wa, lo_ba; // per-layer block: W_p^T, taps [lo+ro][proj], W_a^T, b_a
  // training forward only (fsmn_train_kernel): the activations the backward needs, one (B * save_T, width) block per
  // activation in the order of fsmn_saved_offset; this chunk's frames start at save_t0 of each utterance's save_T
  float* saved;
  int save_T, save_t0;
};

// The saved activations of a training forward over M = B * T frames, as consecutive (M, width) row-major blocks:
//   x1 (aff_in), h0 (lin), then per layer l: p_l (proj), m_l (proj), h_{l+1} (lin), then x5 (aff_out).
// Floats per frame: aff_in + lin + L * (2 proj + lin) + aff_out.  which: 0 x1, 1 h0, 2 p_l, 3 m_l, 4 h_{l+1}, 5 x5.
__host__ __device__ inline long long fsmn_saved_offset(const FsmnArgs& a, long long M, int which, int l) {
  const long long per_layer = 2LL * a.proj + a.lin, head = (long long)a.aff_in + a.lin;
  switch (which) {
    case 0: return 0;
    case 1: return M * a.aff_in;
    case 2: return M * (head + l * per_layer);
    case 3: return M * (head + l * per_layer + a.proj);
    case 4: return M * (head + l * per_layer + 2LL * a.proj);
    default: return M * (head + a.L * per_layer);
  }
}
inline long long fsmn_saved_per_frame(const FsmnArgs& a) {
  return (long long)a.aff_in + a.lin + (long long)a.L * (2LL * a.proj + a.lin) + a.aff_out;
}

size_t fsmn_smem_bytes(const FsmnArgs& a);
int fsmn_tile_rows();
int fsmn_pass_cols();
int fsmn_launch(FsmnArgs a, cudaStream_t st);
int fsmn_train_launch(FsmnArgs a, cudaStream_t st);    // fsmn_launch that also stores a.saved

// fsmn_grad.cu -------------------------------------------------------------------------------------------------------
constexpr int FSMN_MAX_LAYERS = 16;
constexpr int FSMN_MAX_TAPS = 32;                          // lorder + rorder: one register per tap in the memory kernel
constexpr int FSMN_MAX_PARAMS = 8 + 5 * FSMN_MAX_LAYERS;   // parameters of an FSMN of L layers: 8 + 5 L
constexpr int FSMN_GRAD_SLICES = 32;                       // row slices of every weight-gradient reduction

// One parameter tensor of the state_dict: src viewed as [rows][cols] lands transposed at packed[dst + c * ld + r]
// (a Linear weight [N][K] -> W^T [K][Npad]; a bias: cols 1; a tap bank [proj][order] -> [order][proj]).  The host
// pack of the FSMN and GRU models (model_host.cu place) writes every parameter by this rule and keeps each one's
// dst, rows, cols and ld, so the device pack of wekws_model_load_params reuses the host's layout.
struct FsmnParamCopy {
  const float* src;
  long long dst;
  int rows, cols, ld;
};
struct FsmnPackArgs {
  float* packed;
  int n;
  FsmnParamCopy p[FSMN_MAX_PARAMS];
};
int fsmn_pack_launch(const FsmnPackArgs& a, cudaStream_t st);

// Backward of a training forward: rows M = B * T, every frame (padding included).  grads[i] in the parameter order of
// the pack (state_dict order).  Workspace: fsmn_backward_workspace_floats(a, M) floats.
long long fsmn_backward_workspace_floats(const FsmnArgs& a, long long M);
int fsmn_backward_launch(const FsmnArgs& a, const float* feats, const float* saved, const float* grad_out, int B, int T,
                         float* const* grads, float* workspace, cudaStream_t st);
int fsmn_backward_launches(int L);

}  // namespace wekws
