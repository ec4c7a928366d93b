// Kernel argument block of the fused convolutional-backbone kernel (conv_backbone.cu).
#pragma once
#include <cuda_runtime.h>

namespace wekws {

constexpr int kMaxBlocks = 40;

struct ConvArgs {
  // tensors
  const float* feats;      // (B, T, idim)
  const float* in_cache;   // (B, C, P) or nullptr
  float* out;              // (B, T, odim)
  float* out_cache;        // (B, C, P)
  const float* wstream;    // GEMM weight chunks in consumption order, each [rows][C]
  const int* chunk_off;    // n_chunks + 1 prefix offsets (floats) into wstream
  const float* vec;        // per-channel vectors + classifier
  // model
  int kind;                // wekws_backbone
  int C, idim, odim, nblocks, ktaps, P, stack_size, act, has_cmvn;
  int n_chunks;
  int v_mean, v_istd, v_bp, v_blocks, v_blk_stride, v_wc, v_bc;
  int dil[kMaxBlocks];
  int coff[kMaxBlocks];
  // call
  int B, T;
  long long feat_bstride, out_bstride;   // floats between consecutive streams in feats / out
  // derived by conv_backbone_launch
  int S, RP, PADMAX, KP, ah_floats, n_tiles;
  // utterance-level head (cls_head.cu): pool != nullptr replaces the per-frame classifier by the per-stream sum of the
  // classifier input over frames [pool_t0, pool_t1) of this chunk, stored to pool (B, C) (pool_add = 0) or added to it
  float* pool;
  int pool_t0, pool_t1, pool_add;
};

int conv_chunk_rows(int C);
int conv_backbone_launch(ConvArgs a, int padmax_raw, cudaStream_t st);
// Largest chunk length T one CTA can hold (S = 1).
int conv_backbone_max_T(const ConvArgs& a, int padmax_raw);

}  // namespace wekws
