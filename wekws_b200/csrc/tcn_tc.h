// Kernel argument block of the tensor-core dense-TCN kernel (tcn_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_backbone.h"

namespace wekws {

struct TcnTcArgs {
  const float* feats;      // (B, T, idim), stream stride feat_bstride
  const float* in_cache;   // (B, 64, P) or nullptr
  float* out;              // (B, T, odim), stream stride out_bstride
  float* out_cache;        // (B, 64, P)
  const uint8_t* wimg;     // 16 KB bf16 hi|lo images: [Wp atom0][Wp atom1][blk0 tap0]..[blk0 tapK-1][blk1 tap0]...
  const float* vec;        // same per-channel vector blob as the FFMA kernel
  int B, T;
  long long feat_bstride, out_bstride;
  int idim, odim, nblocks, ktaps, P, act, has_cmvn;
  int v_mean, v_istd, v_bp, v_blocks, v_blk_stride, v_wc, v_bc;
  int dil[kMaxBlocks];
  int coff[kMaxBlocks];
  int smax, spt, padr;     // streams per pass / per tile, roundup4(max pad) (set by tcn_tc_launch)
};

bool tcn_tc_eligible(const TcnTcArgs& a, int padmax);
int tcn_tc_max_T(int padmax);   // chunk height: 128 frames, fewer when the pad leaves less room in the tile
int tcn_tc_launch(TcnTcArgs a, int padmax, cudaStream_t st);

}  // namespace wekws
