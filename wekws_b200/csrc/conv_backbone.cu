// Fused whole-network kernel for the convolutional WeKws backbones (FP32 FMA path).
//
// One launch computes, for a chunk of T frames of B independent streams,
//   CMVN -> Linear+ReLU -> every causal dilated block (MDTC / DS-TCN / TCN) -> classifier
//   -> activation, and the new streaming cache -- i.e. all of KWSModel.forward
// (reference wekws/model/kws_model.py:65-76; blocks mdtc.py:95-121, tcn.py:35-61) with
// every eval-mode BatchNorm pre-folded into its producer by model_host.cu.
//
// Work decomposition: a CTA owns a tile of S whole streams (ROWS = S*T frames) and walks
// the network layer by layer with the residual stream resident in shared memory,
// channel-major / time-minor (the reference cache layout, so cache segments copy
// straight in and out):
//     xbuf[C][RP]  residual stream x            abuf[C][RP]  depthwise output / tap copy
//     hbuf[C][RP]  pointwise-1 output           halo[C][S][PADMAX]  this block's cache slice
//     ring[2][SLOT] double-buffered weight chunks streamed from L2 with cp.async
// Each cache byte is read once (cp.async, one block ahead) and written once.
// GEMMs are register-tiled FP32 FFMA: a thread owns 4 output channels x 4*TPT frames.
#include "common.cuh"
#include "conv_backbone.h"

namespace wekws {

namespace {

constexpr int NT = 512;          // threads per CTA (16 warps)
constexpr int TPT = 2;           // row passes per thread in the GEMM tile map

struct AsyncGroups {
  int committed = 0;
  __device__ __forceinline__ int commit() { cp_async_commit(); return ++committed; }
  __device__ __forceinline__ void wait(int seq) { cp_async_wait_pending(committed - seq); }
};

template <int C>
struct WPipe {
  static constexpr int KC = (C <= 128) ? 64 : 32;   // weight rows per chunk
  static constexpr int SLOT = KC * C;               // floats per ring slot
  float* ring;
  const float* g;
  const int* off;
  int n;
  int seq_issued = 0, seq_cur = 0;
  int grp[2] = {0, 0};

  __device__ __forceinline__ void issue(AsyncGroups& ag) {
    const int chunk = seq_issued % n;
    const int slot = seq_issued & 1;
    const int beg = __ldg(off + chunk), end = __ldg(off + chunk + 1);
    float* dst = ring + slot * SLOT;
    const float* src = g + beg;
    for (int i = threadIdx.x * 4; i < end - beg; i += NT * 4) cp_async16(dst + i, src + i);
    grp[slot] = ag.commit();
    ++seq_issued;
  }
  // Returns the smem pointer of the current chunk; prefetches the following one.
  __device__ __forceinline__ const float* acquire(AsyncGroups& ag) {
    const int slot = seq_cur & 1;
    ag.wait(grp[slot]);
    __syncthreads();
    issue(ag);
    ++seq_cur;
    return ring + slot * SLOT;
  }
};

template <int C>
struct TileMap {
  int o0;            // first of this thread's 4 output channels
  int r0[TPT];       // first of 4 rows, per pass
  bool valid[TPT];
  __device__ __forceinline__ void init(int RP) {
    constexpr int NOGB = C / 32;           // warps side by side along the channel axis
    constexpr int RB = 16 / NOGB;          // 16-row blocks covered per pass by 16 warps
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    const int ogb = w % NOGB, rgb = w / NOGB;
    o0 = (ogb * 8 + (l & 7)) * 4;
#pragma unroll
    for (int t = 0; t < TPT; ++t) {
      r0[t] = 16 * (rgb + t * RB) + 4 * (l >> 3);
      valid[t] = r0[t] < RP;
    }
  }
};

#define FMA16(ACC, W4, A4)                                                             \
  ACC[0] = fmaf(W4.x, A4.x, ACC[0]);   ACC[1] = fmaf(W4.x, A4.y, ACC[1]);              \
  ACC[2] = fmaf(W4.x, A4.z, ACC[2]);   ACC[3] = fmaf(W4.x, A4.w, ACC[3]);              \
  ACC[4] = fmaf(W4.y, A4.x, ACC[4]);   ACC[5] = fmaf(W4.y, A4.y, ACC[5]);              \
  ACC[6] = fmaf(W4.y, A4.z, ACC[6]);   ACC[7] = fmaf(W4.y, A4.w, ACC[7]);              \
  ACC[8] = fmaf(W4.z, A4.x, ACC[8]);   ACC[9] = fmaf(W4.z, A4.y, ACC[9]);              \
  ACC[10] = fmaf(W4.z, A4.z, ACC[10]); ACC[11] = fmaf(W4.z, A4.w, ACC[11]);            \
  ACC[12] = fmaf(W4.w, A4.x, ACC[12]); ACC[13] = fmaf(W4.w, A4.y, ACC[13]);            \
  ACC[14] = fmaf(W4.w, A4.z, ACC[14]); ACC[15] = fmaf(W4.w, A4.w, ACC[15]);

// acc[t][i*4+j] += sum_k W[k][o0+i] * A[k][r0[t]+j]     (A channel-major: [K][RP])
// RP is a multiple of 16, so a warp's four row groups are valid or padding together (no divergence).
template <int C, bool TWO>
__device__ __forceinline__ void gemm_cm_impl(float (&acc)[TPT][16], const float* __restrict__ A, int RP,
                                             const float* __restrict__ W, int K, const TileMap<C>& tm) {
  const float* wp = W + tm.o0;
  const float* a0 = A + tm.r0[0];
  const float* a1 = A + tm.r0[1];
#pragma unroll 8
  for (int k = 0; k < K; ++k) {
    const float4 w4 = *reinterpret_cast<const float4*>(wp);
    wp += C;
    const float4 x0 = *reinterpret_cast<const float4*>(a0);
    a0 += RP;
    FMA16(acc[0], w4, x0)
    if (TWO) {
      const float4 x1 = *reinterpret_cast<const float4*>(a1);
      a1 += RP;
      FMA16(acc[1], w4, x1)
    }
  }
}
template <int C>
__device__ __forceinline__ void gemm_cm(float (&acc)[TPT][16], const float* __restrict__ A, int RP,
                                        const float* __restrict__ W, int K, const TileMap<C>& tm) {
  if (tm.valid[1]) gemm_cm_impl<C, true>(acc, A, RP, W, K, tm);
  else if (tm.valid[0]) gemm_cm_impl<C, false>(acc, A, RP, W, K, tm);
}

// Same with A row-major: A[r][KP] (first Linear: frames x idim), column offset k0.
template <int C, bool TWO>
__device__ __forceinline__ void gemm_rm_impl(float (&acc)[TPT][16], const float* __restrict__ A, int KP,
                                             const float* __restrict__ W, int K, const TileMap<C>& tm) {
  const float* wp = W + tm.o0;
  const float* a0 = A + tm.r0[0] * KP;
  const float* a1 = A + tm.r0[1] * KP;
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const float4 w4 = *reinterpret_cast<const float4*>(wp);
    wp += C;
    float4 x0;
    x0.x = a0[k]; x0.y = a0[KP + k]; x0.z = a0[2 * KP + k]; x0.w = a0[3 * KP + k];
    FMA16(acc[0], w4, x0)
    if (TWO) {
      float4 x1;
      x1.x = a1[k]; x1.y = a1[KP + k]; x1.z = a1[2 * KP + k]; x1.w = a1[3 * KP + k];
      FMA16(acc[1], w4, x1)
    }
  }
}
template <int C>
__device__ __forceinline__ void gemm_rm(float (&acc)[TPT][16], const float* __restrict__ A, int KP,
                                        const float* __restrict__ W, int K, const TileMap<C>& tm) {
  if (tm.valid[1]) gemm_rm_impl<C, true>(acc, A, KP, W, K, tm);
  else if (tm.valid[0]) gemm_rm_impl<C, false>(acc, A, KP, W, K, tm);
}

__device__ __forceinline__ void zero_acc(float (&acc)[TPT][16]) {
#pragma unroll
  for (int t = 0; t < TPT; ++t)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[t][i] = 0.f;
}

__device__ __forceinline__ float4 relu4(float4 v) {
  return make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
}
__device__ __forceinline__ float4 add4(float4 a, float4 b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}

enum { EPI_RELU_STORE = 0,      // dst = relu(acc + b)
       EPI_MDTC_OUT = 1,        // dst = relu(acc + b + x)            (x == dst, in place)
       EPI_TCN_OUT = 2 };       // dst = relu(acc + b) + x            (x == dst, in place)

template <int C, int MODE>
__device__ __forceinline__ void epilogue(const float (&acc)[TPT][16], const float* __restrict__ bias,
                                         float* __restrict__ dst, int RP, const TileMap<C>& tm,
                                         float (*msum)[16], bool add_msum) {
  const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + tm.o0));
  const float bb[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
  for (int t = 0; t < TPT; ++t) {
    if (!tm.valid[t]) continue;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      float* p = dst + (tm.o0 + i) * RP + tm.r0[t];
      float4 v = make_float4(acc[t][i * 4 + 0] + bb[i], acc[t][i * 4 + 1] + bb[i],
                             acc[t][i * 4 + 2] + bb[i], acc[t][i * 4 + 3] + bb[i]);
      if (MODE == EPI_RELU_STORE) {
        v = relu4(v);
      } else if (MODE == EPI_MDTC_OUT) {
        v = relu4(add4(v, *reinterpret_cast<const float4*>(p)));
      } else {
        v = add4(relu4(v), *reinterpret_cast<const float4*>(p));
      }
      *reinterpret_cast<float4*>(p) = v;
      if (MODE == EPI_MDTC_OUT && add_msum) {
        msum[t][i * 4 + 0] += v.x; msum[t][i * 4 + 1] += v.y;
        msum[t][i * 4 + 2] += v.z; msum[t][i * 4 + 3] += v.w;
      }
    }
  }
}

// Value of cat(cache_slice, x) of stream s, channel c at cat position p (0 <= p < pad + T).
__device__ __forceinline__ float cat_at(const float* __restrict__ xrow, const float* __restrict__ hrow,
                                        int s, int T, int pad, int p) {
  return p < pad ? hrow[p] : xrow[s * T + p - pad];
}

template <int C>
__global__ void __launch_bounds__(NT, 1) conv_backbone_kernel(const ConvArgs a) {
  extern __shared__ __align__(16) float smem[];
  const int RP = a.RP, S = a.S, T = a.T, PADMAX = a.PADMAX;
  float* xbuf = smem;
  float* abuf = xbuf + C * RP;                 // region AH starts here (fin aliases it)
  float* hbuf = abuf + C * RP;
  float* halo = abuf + a.ah_floats;
  float* ring = halo + C * S * PADMAX;
  float* fin = abuf;                           // [RP][KP] row-major input features

  TileMap<C> tm;
  tm.init(RP);
  AsyncGroups ag;
  WPipe<C> wp;
  wp.ring = ring; wp.g = a.wstream; wp.off = a.chunk_off; wp.n = a.n_chunks;
  wp.issue(ag);                                // chunk 0 of the first tile

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int K = a.ktaps;
  const float* vec = a.vec;

  for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const int b0 = tile * S;
    const int Sv = min(S, a.B - b0);           // valid streams in this tile
    const int ROWS = Sv * T;
    // rows owned by this lane in the time-parallel loops: r = lane + 32*qi  ->  (stream, frame); -1 = padding row
    int row_s[8], row_t[8];
#pragma unroll
    for (int qi = 0; qi < 8; ++qi) {
      const int r = lane + 32 * qi;
      const int sidx = r / T;
      row_s[qi] = r < ROWS ? sidx : -1;
      row_t[qi] = r - sidx * T;
    }

    // issue the cache slice of block `blk` into halo (zero when no cache / invalid stream)
    auto issue_halo = [&](int blk) -> int {
      const int pad = a.dil[blk] * (K - 1), off = a.coff[blk];
      const int n = C * S * pad;
      for (int idx = tid; idx < n; idx += NT) {
        const int j = idx % pad, cs = idx / pad, c = cs % C, s = cs / C;
        float* dst = halo + (c * S + s) * PADMAX + j;
        if (a.in_cache != nullptr && s < Sv)
          cp_async4(dst, a.in_cache + ((size_t)(b0 + s) * C + c) * a.P + off + j);
        else
          *dst = 0.f;
      }
      return ag.commit();
    };

    // ---- stage 0: features -> fin[r][KP] with CMVN applied; halo of block 0 in flight ----
    __syncthreads();                           // previous tile fully done with smem
    int hgrp = issue_halo(0);
    {
      const int idim = a.idim, KP = a.KP;
      for (int idx = tid; idx < RP * idim; idx += NT) {
        const int r = idx / idim, k = idx - r * idim;
        float v = 0.f;
        if (r < ROWS) {
          const int s = r / T, t = r - s * T;
          v = __ldg(a.feats + (size_t)(b0 + s) * a.feat_bstride + (size_t)t * idim + k);
          if (a.has_cmvn) v = (v - __ldg(vec + a.v_mean + k)) * __ldg(vec + a.v_istd + k);
        }
        fin[r * KP + k] = v;
      }
    }
    float acc[TPT][16];
    float msum[TPT][16];
    zero_acc(acc);
    zero_acc(msum);
    for (int k0 = 0; k0 < a.idim; k0 += WPipe<C>::KC) {
      const float* W = wp.acquire(ag);         // (sync inside: fin visible)
      gemm_rm<C>(acc, fin + k0, a.KP, W, min(WPipe<C>::KC, a.idim - k0), tm);
    }
    __syncthreads();                           // everyone done reading fin (aliases abuf/hbuf)
    epilogue<C, EPI_RELU_STORE>(acc, vec + a.v_bp, xbuf, RP, tm, msum, false);

    // ---- blocks ----
    for (int blk = 0; blk < a.nblocks; ++blk) {
      const int d = a.dil[blk], pad = d * (K - 1), off = a.coff[blk];
      const float* vb = vec + a.v_blocks + blk * a.v_blk_stride;
      ag.wait(hgrp);
      __syncthreads();                         // halo landed; xbuf complete

      // new cache slice: last `pad` columns of cat(cache, x)       (mdtc.py:113 / tcn.py:54)
      {
        const int n = C * Sv * pad;
        for (int idx = tid; idx < n; idx += NT) {
          const int j = idx % pad, cs = idx / pad, c = cs % C, s = cs / C;
          const float v = cat_at(xbuf + c * RP, halo + (c * S + s) * PADMAX, s, T, pad, T + j);
          a.out_cache[((size_t)(b0 + s) * C + c) * a.P + off + j] = v;
        }
      }

      if (a.kind == WEKWS_BACKBONE_TCN) {
        // dense dilated conv: K accumulating GEMMs, tap j reads cat shifted by j*d
        zero_acc(acc);
        for (int j = 0; j < K; ++j) {
          float* buf = (j & 1) ? hbuf : abuf;
          for (int c = warp; c < C; c += NT / 32) {
            const float* xrow = xbuf + c * RP;
#pragma unroll
            for (int qi = 0; qi < 8; ++qi) {
              const int r = lane + 32 * qi;
              if (r < RP) {
                float v = 0.f;
                if (row_s[qi] >= 0)
                  v = cat_at(xrow, halo + (c * S + row_s[qi]) * PADMAX, row_s[qi], T, pad, row_t[qi] + j * d);
                buf[c * RP + r] = v;
              }
            }
          }
          for (int k0 = 0; k0 < C; k0 += WPipe<C>::KC) {
            const float* W = wp.acquire(ag);   // sync inside publishes buf
            // after the last tap's copy nobody reads halo any more: prefetch the next slice
            if (j == K - 1 && k0 == 0 && blk + 1 < a.nblocks) hgrp = issue_halo(blk + 1);
            gemm_cm<C>(acc, buf + k0 * RP, RP, W, WPipe<C>::KC < C ? WPipe<C>::KC : C, tm);
          }
        }
        epilogue<C, EPI_TCN_OUT>(acc, vb, xbuf, RP, tm, msum, false);
      } else {
        // depthwise dilated conv (+folded BN; ReLU for DS-TCN)     (mdtc.py:56-57 / tcn.py:102-109)
        const bool dw_relu = (a.kind == WEKWS_BACKBONE_DSTCN);
        for (int c = warp; c < C; c += NT / 32) {
          float wt[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) wt[j] = j < K ? __ldg(vb + j * C + c) : 0.f;
          const float bias = __ldg(vb + K * C + c);
          const float* xrow = xbuf + c * RP;
#pragma unroll
          for (int qi = 0; qi < 8; ++qi) {
            const int r = lane + 32 * qi;
            if (r < RP) {
              float v = 0.f;
              if (row_s[qi] >= 0) {
                const int sidx = row_s[qi], t = row_t[qi];
                const float* hrow = halo + (c * S + sidx) * PADMAX;
                v = bias;
#pragma unroll
                for (int j = 0; j < 8; ++j)
                  if (j < K) v = fmaf(wt[j], cat_at(xrow, hrow, sidx, T, pad, t + j * d), v);
                if (dw_relu) v = fmaxf(v, 0.f);
              }
              abuf[c * RP + r] = v;
            }
          }
        }
        const float* vb1 = vb + (K + 1) * C;
        zero_acc(acc);
        bool first = true;
        for (int k0 = 0; k0 < C; k0 += WPipe<C>::KC) {
          const float* W = wp.acquire(ag);     // sync inside: abuf visible, halo free
          if (first && blk + 1 < a.nblocks) hgrp = issue_halo(blk + 1);
          first = false;
          gemm_cm<C>(acc, abuf + k0 * RP, RP, W, WPipe<C>::KC < C ? WPipe<C>::KC : C, tm);
        }
        if (a.kind == WEKWS_BACKBONE_DSTCN) {
          epilogue<C, EPI_TCN_OUT>(acc, vb1, xbuf, RP, tm, msum, false);
        } else {
          epilogue<C, EPI_RELU_STORE>(acc, vb1, hbuf, RP, tm, msum, false);
          zero_acc(acc);
          for (int k0 = 0; k0 < C; k0 += WPipe<C>::KC) {
            const float* W = wp.acquire(ag);   // sync inside: hbuf visible
            gemm_cm<C>(acc, hbuf + k0 * RP, RP, W, WPipe<C>::KC < C ? WPipe<C>::KC : C, tm);
          }
          const bool stack_end = (blk > 0) && (blk % a.stack_size == 0);
          epilogue<C, EPI_MDTC_OUT>(acc, vb1 + C, xbuf, RP, tm, msum, stack_end);
        }
      }
    }

    // ---- classifier + activation ----
    const float* cls_in = xbuf;
    if (a.kind == WEKWS_BACKBONE_MDTC) {       // multi-scale sum of the stack outputs (mdtc.py:270-273)
      __syncthreads();
#pragma unroll
      for (int t = 0; t < TPT; ++t) {
        if (!tm.valid[t]) continue;
#pragma unroll
        for (int i = 0; i < 4; ++i)
          *reinterpret_cast<float4*>(abuf + (tm.o0 + i) * RP + tm.r0[t]) =
              make_float4(msum[t][i * 4], msum[t][i * 4 + 1], msum[t][i * 4 + 2], msum[t][i * 4 + 3]);
      }
      cls_in = abuf;
    }
    __syncthreads();
    if (a.pool != nullptr) {
      // utterance-level head (cls_head.cu): per-stream sum of the classifier input over frames [pool_t0, pool_t1), one
      // warp per (stream, channel): lane-strided frames, then a butterfly in a fixed order; the first time-chunk of the
      // call stores, later ones add
      if (a.pool_t1 > a.pool_t0) {
        for (int idx = warp; idx < Sv * C; idx += NT / 32) {
          const int s = idx / C, c = idx - s * C;
          const float* src = cls_in + c * RP + s * T;
          float v = 0.f;
          for (int t = a.pool_t0 + lane; t < a.pool_t1; t += 32) v += src[t];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
          if (lane == 0) {
            float* g = a.pool + (size_t)(b0 + s) * C + c;
            *g = a.pool_add ? *g + v : v;
          }
        }
      }
    } else {
      const int odim = a.odim;
      const float* wc = vec + a.v_wc;          // [C][odim]  (transposed classifier weight)
      for (int idx = tid; idx < ROWS * odim; idx += NT) {
        const int r = idx / odim, j = idx - r * odim;
        const int s = r / T, t = r - s * T;
        float y = __ldg(vec + a.v_bc + j);
#pragma unroll 8
        for (int c = 0; c < C; ++c) y = fmaf(__ldg(wc + c * odim + j), cls_in[c * RP + r], y);
        if (a.act == WEKWS_ACT_SIGMOID) y = sigmoidf_acc(y);
        a.out[(size_t)(b0 + s) * a.out_bstride + (size_t)t * odim + j] = y;
      }
    }
  }
  cp_async_wait_pending(0);                    // drain the speculative prefetch of the next chunk
}

template <int C>
int launch_c(const ConvArgs& a, int grid, size_t smem, cudaStream_t st) {
  if (const int rc = opt_in_smem((const void*)conv_backbone_kernel<C>, smem)) return rc;
  conv_backbone_kernel<C><<<grid, NT, smem, st>>>(a);
  return check_launch("conv_backbone_kernel");
}

}  // namespace

int conv_chunk_rows(int C) { return C <= 128 ? 64 : 32; }

namespace {
constexpr size_t kSmemCap = 227 * 1024;

// rows a tile may hold: what the GEMM tile map covers, capped at the 8 x 32 rows the time-parallel loops
// (row_s / row_t, depthwise conv, tap copies) walk -- hidden 32 would otherwise map 512 rows
int max_rows_map(int C) {
  const int m = 16 * (16 / (C / 32)) * TPT;
  return m < 256 ? m : 256;
}

// Shared-memory bytes of a tile of S streams / RP padded rows; *ah = floats of region AH.
size_t tile_smem(const ConvArgs& a, int S, int RP, int PADMAX, int KP, size_t* ah) {
  const int C = a.C;
  const int nbuf = (a.kind == WEKWS_BACKBONE_DSTCN) ? 2 : 3;   // xbuf + abuf (+ hbuf)
  size_t ahf = (size_t)(nbuf - 1) * C * RP;
  const size_t fin = (size_t)RP * KP;
  if (fin > ahf) ahf = fin;
  ahf = (ahf + 3) & ~(size_t)3;
  *ah = ahf;
  return ((size_t)C * RP + ahf + (size_t)C * S * PADMAX + 2 * (size_t)conv_chunk_rows(C) * C) * sizeof(float);
}
}  // namespace

int conv_backbone_max_T(const ConvArgs& a, int padmax_raw) {
  const int KP = a.idim | 1;
  int best = 0;
  for (int T = 1; T <= max_rows_map(a.C); ++T) {
    size_t ah;
    const int RP = (T + 15) & ~15;
    if (RP > max_rows_map(a.C) || tile_smem(a, 1, RP, padmax_raw, KP, &ah) > kSmemCap) break;
    best = T;
  }
  return best;
}

// Chooses the tile shape for (B, T), fills the derived fields of `a` and launches.
int conv_backbone_launch(ConvArgs a, int padmax_raw, cudaStream_t st) {
  const int C = a.C;
  WEKWS_REQUIRE(C == 32 || C == 64 || C == 128 || C == 256, "hidden_dim %d unsupported (32/64/128/256)", C);
  WEKWS_REQUIRE(a.T >= 1 && a.B >= 1, "conv_backbone_launch: empty call");
  a.PADMAX = padmax_raw;
  a.KP = a.idim | 1;                           // odd row stride -> conflict-free strided reads
  // largest S that fits the tile map and shared memory
  int smax = 0;
  for (int S = 1; S <= a.B; ++S) {
    const int RP = (S * a.T + 15) & ~15;
    size_t ah;
    if (RP > max_rows_map(C) || tile_smem(a, S, RP, a.PADMAX, a.KP, &ah) > kSmemCap) break;
    smax = S;
  }
  WEKWS_REQUIRE(smax >= 1, "chunk of T=%d frames does not fit one CTA (hidden_dim %d)", a.T, C);
  // pick S minimising (waves x padded rows per tile): balances the SMs for small batches
  const int sms = device_sm_count();
  int best = smax;
  long best_cost = -1;
  for (int S = 1; S <= smax; ++S) {
    const long tiles = (a.B + S - 1) / S;
    const long waves = (tiles + sms - 1) / sms;
    const long cost = waves * ((((long)S * a.T + 15) & ~15L) + 24);   // +24: fixed per-tile overhead in row units
    if (best_cost < 0 || cost <= best_cost) { best_cost = cost; best = S; }
  }
  a.S = best;
  a.RP = (a.S * a.T + 15) & ~15;
  size_t ah;
  const size_t smem = tile_smem(a, a.S, a.RP, a.PADMAX, a.KP, &ah);
  a.ah_floats = (int)ah;
  a.n_tiles = (a.B + a.S - 1) / a.S;
  const int grid = a.n_tiles < sms ? a.n_tiles : sms;
  switch (C) {
    case 32: return launch_c<32>(a, grid, smem, st);
    case 64: return launch_c<64>(a, grid, smem, st);
    case 128: return launch_c<128>(a, grid, smem, st);
    default: return launch_c<256>(a, grid, smem, st);
  }
}

}  // namespace wekws
