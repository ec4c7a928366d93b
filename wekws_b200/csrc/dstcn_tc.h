// Kernel argument block of the tensor-core depthwise-separable TCN kernel (dstcn_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_backbone.h"

namespace wekws {

struct DsTcArgs {
  const float* feats;      // (B, T, idim), stream stride feat_bstride
  const float* in_cache;   // (B, 256, P) or nullptr
  float* out;              // (B, T, odim), stream stride out_bstride
  float* out_cache;        // (B, 256, P); may alias in_cache
  const uint8_t* wimg;     // 32 KB bf16 hi|lo images of 128 output channels x 64 K:
                           //   [Wp atom0 half0][atom0 half1]([atom1 half0][atom1 half1])
                           //   then per block, per 64-channel K slab ks: [ks half0][ks half1]
  const float* vec;        // same per-channel vector blob as the FFMA kernel
  int B, T;
  long long feat_bstride, out_bstride;
  int idim, odim, nblocks, ktaps, P, act, has_cmvn;
  int v_mean, v_istd, v_bp, v_blocks, v_blk_stride, v_wc, v_bc;
  int dil[kMaxBlocks];
  int coff[kMaxBlocks];
  int spt;                 // streams per 128-row tile (set by dstcn_tc_launch)
  int aliased;             // out_cache overlaps in_cache (set by dstcn_tc_launch)
  float* hidden;           // non-null: skip the classifier and write the final x as (B, T, 256) rows (stream stride
  long long hidden_bstride;  // hidden_bstride) for the tensor-core classifier (linear_tc.cu) that follows
};

// cls_gemm: the classifier runs as its own GEMM (linear_tc.cu) on `hidden`, so odim is not limited
bool dstcn_tc_eligible(const DsTcArgs& a, int hdim, bool cls_gemm);
int dstcn_tc_max_T();
int dstcn_tc_launch(DsTcArgs a, cudaStream_t st);

}  // namespace wekws
