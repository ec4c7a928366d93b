// Kernel argument block of the tensor-core MDTC kernel (mdtc_tc.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "conv_backbone.h"

namespace wekws {

constexpr int kTcMaxBlocks = 17;   // 17 x 7 x 256 B = 30464 B of the 32764-byte parameter block (mdtc: 1 + 4 x 4)

struct TcArgs {
  const float* feats;      // (B, T, idim), stream stride feat_bstride
  const float* in_cache;   // (B, 64, P) or nullptr
  float* out;              // (B, T, odim), stream stride out_bstride
  float* out_cache;        // (B, 64, P)
  const uint8_t* wimg;     // pre-swizzled bf16 hi|lo weight images, 16 KB per slot:
                           //   [Wp atom0][Wp atom1][blk0 W1][blk0 W2][blk1 W1]...
  const float* vec;        // same per-channel vector blob as the FFMA kernel
  int B, T;
  long long feat_bstride, out_bstride;
  int idim, odim, nblocks, ktaps, P, stack_size, act, has_cmvn;
  int v_mean, v_istd, v_bp, v_blocks, v_blk_stride, v_wc, v_bc;
  int dil[kMaxBlocks];
  int coff[kMaxBlocks];
  int smax, spt, padr;     // streams per pass / per tile, roundup4(max pad) (set by mdtc_tc_launch)
  int tmap_idx[kMaxBlocks];               // block -> tensor map (one per distinct pad)
  alignas(64) CUtensorMap tmap[4];        // 2-D maps over in_cache viewed as [B*64][P], box [64][pad]
  // Per-block depthwise taps and the two GEMM biases, passed BY VALUE in the kernel parameter block (constant bank), so
  // they never touch the shared-memory load/store pipe.  [blk][0..4] = taps (zero beyond ktaps), [5] = b1, [6] = b2;
  // 64 each.
  alignas(16) float4 cw[kTcMaxBlocks][7 * 16];
  // head variant of the kernel only (cls_head.cu): per-stream sum of the stack-output sum over frames
  // [pool_t0, pool_t1) of this chunk, stored to pool (B, 64) (pool_add = 0) or added to it
  float* pool;
  int pool_t0, pool_t1, pool_add;
};
static_assert(sizeof(TcArgs) <= 32764, "kernel parameter block exceeds 32764 bytes");

// head: the utterance-level head variant (a.pool set; no per-frame output, so no limit on odim)
bool tc_eligible(const TcArgs& a, int padmax, bool head = false);
int tc_max_T();
int mdtc_tc_launch(TcArgs a, int padmax, cudaStream_t st, bool head = false);

}  // namespace wekws
