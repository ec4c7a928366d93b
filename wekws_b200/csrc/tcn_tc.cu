// Tensor-core (wgmma) fused forward for the dense TCN backbone with hidden_dim 64
// (reference wekws/model/tcn.py:67-88 CnnBlock inside TCN :122-166; BatchNorm folded):
//     per block:  o = ReLU( sum_j W_j . cat(cache, x)[:, t + j*d] + b ) ;  x' = o + x
// i.e. a K-tap dilated convolution = K accumulating 64x64 GEMMs whose A operand is the residual stream
// shifted by j*d frames.  All streams of a CTA stay resident in shared memory (X[c][col], cache slice in front of
// each stream's frames so a tap is a column offset); bf16x3 split; every warpgroup owns 64 rows of one of the two
// 128-row tiles, builds the A fragment of each tap straight from X into registers and accumulates the taps in a
// register accumulator (wgmma m64n64k16, A from registers); weights are pre-swizzled 16 KB images streamed through
// a 4-slot ring by cp.async.bulk.  TCN cache rows are 105 floats and slices 7..56 floats wide -- not 16-byte
// multiples, so TMA cannot fetch them: the compute warps use 4-byte cp.async straight into X instead.
#include <stdlib.h>

#include "common.cuh"
#include "tc_common.cuh"
#include "tcn_tc.h"

namespace wekws {

namespace {

using namespace tc;

constexpr int NCW = 16, NCT = NCW * 32, NT_TC = NCT + 32;
constexpr int C = 64;
constexpr int NTILE = 2;
constexpr int RPX = 512, XCOLS = 504;
constexpr int X_BYTES = 64 * RPX * 4;
constexpr int W_SLOT = 16384, NW = 4;
constexpr int OFF_X = 0, OFF_W = X_BYTES;
constexpr int SMEM_TOTAL = OFF_W + NW * W_SLOT + 1024;            // 197632

__device__ __forceinline__ void compute_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(NCT) : "memory"); }

__global__ void __launch_bounds__(NT_TC, 1) tcn_tc_kernel(const TcnTcArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
  __shared__ uint64_t h_free, w_bar[NW], w_free[NW];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = a.T, K = a.ktaps;
  const float* vec = a.vec;
  float* X = reinterpret_cast<float*>(base + OFF_X);
  uint8_t* Wring = base + OFF_W;
  const uint32_t sbase = smem_u32(base);

  if (tid == 0) {
    mbar_init(&h_free, NCW);
    for (int i = 0; i < NW; ++i) { mbar_init(&w_bar[i], 1); mbar_init(&w_free[i], NCW); }
    mbar_fence_init();
  }
  __syncthreads();
  uint32_t hf_par = 0;
  uint32_t witem = 0;                              // weight items loaded (loader) / consumed (compute) so far
  const int natoms = (a.idim + 63) / 64;
  const int PADR = a.padr, Lw = a.padr + ((T + 3) & ~3);
  const int spt = a.spt;
  const int nitems = 2 + a.nblocks * K;             // weight images per pass: Wp atom 0, atom 1, then the taps

  const int sb = (int)(((long long)a.B * blockIdx.x) / gridDim.x);
  const int se = (int)(((long long)a.B * (blockIdx.x + 1)) / gridDim.x);
  int done = sb;

  while (done < se) {
    const int remaining = se - done;
    const int passes_left = (remaining + a.smax - 1) / a.smax;
    const int ns = (remaining + passes_left - 1) / passes_left;
    const int b0 = done;
    done += ns;
    const int ntile = (ns + spt - 1) / spt;
    auto tile_streams = [&](int i) { return min(spt, ns - i * spt); };

    if (warp == NCW) {
      // ================================================================== WEIGHT RING (lane 0)
      if (lane == 0) {
        for (int n = 0; n < nitems; ++n, ++witem) {
          const uint32_t slot = witem % NW;
          if (witem >= NW) mbar_wait_backoff(&w_free[slot], ((witem / NW) - 1) & 1);
          mbar_arrive_expect_tx(&w_bar[slot], W_SLOT);
          bulk_g2s(Wring + slot * W_SLOT, a.wimg + (size_t)n * W_SLOT, W_SLOT, &w_bar[slot]);
        }
      }
    } else {
      // ================================================================== COMPUTE WARPS
      // warpgroup wgi = warp / 4 owns rows [64 (wgi & 1), +64) of tile wgi / 2 (a warpgroup of an absent tile runs with
      // dead rows only, so that every compute warp consumes every weight image); a thread holds the wgmma fragment of
      // rows r0 and r0 + 8, channel pairs 8 m + 2 (lane % 4)
      const int wgi = warp >> 2, ti = wgi >> 1, q4 = lane & 3;
      const int r0 = 64 * (wgi & 1) + 16 * (warp & 3) + (lane >> 2);
      const int rows_t = ti < ntile ? tile_streams(ti) * T : 0;
      bool live[2];
      int colx[2], sgr[2], ttr[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        live[h] = row < rows_t;
        const int s = live[h] ? row / T : 0;
        sgr[h] = ti * spt + s;
        ttr[h] = live[h] ? row - s * T : 0;
        colx[h] = live[h] ? sgr[h] * Lw + PADR + ttr[h] : XCOLS;
      }
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      uint32_t ahi[4][4], alo[4][4];
      // 3-pass bf16x3 GEMM acc (+)= A * W^T over the next weight image (waited for, released when the MMAs are done)
      auto gemm = [&](int ksteps, bool fresh) {
        const uint32_t slot = witem % NW;
        mbar_wait(&w_bar[slot], (witem / NW) & 1);
        ++witem;
        if (ksteps > 0) {
          const uint64_t dwh = make_sdesc_sw128(sbase + OFF_W + slot * W_SLOT), dwl = dwh + (8192 >> 4);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_rs(acc, ahi[k][0], ahi[k][1], ahi[k][2], ahi[k][3], dwh + 2 * k, (fresh && k == 0) ? 0u : 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_rs(acc, alo[k][0], alo[k][1], alo[k][2], alo[k][3], dwh + 2 * k, 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_rs(acc, ahi[k][0], ahi[k][1], ahi[k][2], ahi[k][3], dwl + 2 * k, 1u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_reg_fence(acc);
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&w_free[slot]);
      };

      // Cache slices of block `blk` -> the pad columns in front of every stream's frames, 4-byte cp.async (rows of the
      // cache are 105 floats, slices 7..56: nothing is 16-byte aligned), spread over ALL compute threads and issued one
      // block ahead, right after the last tap that reads the current block's slices; `halo_wait` + the block barrier
      // publish them.
      auto load_halo = [&](int blk) {
        const int pad = a.dil[blk] * (K - 1), off = a.coff[blk];
        const int per = C * pad;
        for (int e = tid; e < ns * per; e += NCT) {
          const int sg = e / per, r = e - sg * per, c = r / pad, p = r - c * pad;
          float* dst = X + c * RPX + sg * Lw + PADR - pad + p;
          if (a.in_cache) cp_async4(dst, a.in_cache + ((size_t)(b0 + sg) * C + c) * a.P + off + p);
          else *dst = 0.f;
        }
      };
      auto halo_wait = [&]() { asm volatile("cp.async.wait_all;\n" ::: "memory"); };
      // new cache slices (tcn.py:54); afterwards nobody reads the block's cache columns again
      auto store_cache = [&](int blk, int pad) {
        const int off = a.coff[blk];
        for (int i = 0; i < ntile; ++i) {
          const int nst = tile_streams(i), sg0 = i * spt, n = nst * C * pad;
          for (int e = tid; e < n; e += NCT) {
            const int cs = e / pad, j = e - cs * pad, s = cs >> 6, c = cs & 63;
            a.out_cache[((size_t)(b0 + sg0 + s) * C + c) * a.P + off + j] = X[c * RPX + (sg0 + s) * Lw + PADR - pad + T + j];
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&h_free);
      };
      // every compute warp is past the taps (and cache stores) that read the current slices: the columns may be rewritten
      auto halo_free_wait = [&]() {
        mbar_wait(&h_free, hf_par & 1);
        hf_par ^= 1u;
      };

      load_halo(0);                                  // overlaps the feature load and the first Linear
      // ---- features (+CMVN) -> A fragments, first Linear over items 0 (K 0..63) and 1 (K 64..)
      for (int at = 0; at < 2; ++at) {
        if (at < natoms) {
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              const int h = p & 1, kk = 64 * at + 16 * k + 8 * (p >> 1) + 2 * q4;
              float v0 = 0.f, v1 = 0.f;
              if (live[h] && kk < a.idim) {
                const float2 f = __ldg(reinterpret_cast<const float2*>(a.feats + (size_t)(b0 + sgr[h]) * a.feat_bstride +
                                                                       (size_t)ttr[h] * a.idim + kk));
                v0 = f.x; v1 = f.y;
                if (a.has_cmvn) {
                  v0 = (v0 - __ldg(vec + a.v_mean + kk)) * __ldg(vec + a.v_istd + kk);
                  v1 = (v1 - __ldg(vec + a.v_mean + kk + 1)) * __ldg(vec + a.v_istd + kk + 1);
                }
              }
              split2(v0, v1, ahi[k][p], alo[k][p]);
            }
        }
        const int rem = a.idim - 64 * at;
        gemm(at < natoms ? (rem >= 64 ? 4 : (rem + 15) >> 4) : 0, at == 0);
      }
      // ---- x = relu(D + bp) -> X
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(vec + a.v_bp + 8 * j + 2 * q4));
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (live[h]) {
            float* xp = X + (8 * j + 2 * q4) * RPX + colx[h];
            xp[0] = fmaxf(acc[4 * j + 2 * h] + b.x, 0.f);
            xp[RPX] = fmaxf(acc[4 * j + 2 * h + 1] + b.y, 0.f);
          }
      }
      halo_wait();
      compute_barrier();

      for (int blk = 0; blk < a.nblocks; ++blk) {
        const int d = a.dil[blk], pad = d * (K - 1);
        for (int j = 0; j < K; ++j) {
          // The last tap reads frames only (position t + pad), never the cache columns: store the new cache slices
          // and release the columns before it, then fetch the next block's slices while the last tap runs.
          if (j == K - 1) {
            store_cache(blk, pad);
            halo_free_wait();
            if (blk + 1 < a.nblocks) load_halo(blk + 1);
          }
          // tap j: this thread's rows of cat(cache, x) shifted by j*d frames -> A fragments
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              const int h = p & 1, c = 16 * k + 8 * (p >> 1) + 2 * q4;
              const float* xp = X + c * RPX + colx[h] - pad + j * d;
              split2(xp[0], xp[RPX], ahi[k][p], alo[k][p]);
            }
          gemm(4, j == 0);
        }
        compute_barrier();                           // every row's taps have read x
        // x' = relu(D + b) + x -> X                                          (tcn.py:60: no ReLU after the add)
        const float* bb = vec + a.v_blocks + blk * a.v_blk_stride;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(bb + 8 * j + 2 * q4));
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (live[h]) {
              float* xp = X + (8 * j + 2 * q4) * RPX + colx[h];
              xp[0] = fmaxf(acc[4 * j + 2 * h] + b.x, 0.f) + xp[0];
              xp[RPX] = fmaxf(acc[4 * j + 2 * h + 1] + b.y, 0.f) + xp[RPX];
            }
        }
        halo_wait();
        compute_barrier();
      }

      // ---- classifier + activation on x (tcn.py:165 -> classifier.py:63-67)
      const int odim = a.odim;
      for (int i = 0; i < ntile; ++i) {
        const int nrow = tile_streams(i) * T;
        for (int idx = tid; idx < nrow * odim; idx += NCT) {
          const int r = idx / odim, j = idx - r * odim;
          const int s = r / T, tt = r - s * T;
          const float* xc = X + (i * spt + s) * Lw + PADR + tt;
          float y = __ldg(vec + a.v_bc + j);
#pragma unroll 8
          for (int c = 0; c < C; ++c) y = fmaf(__ldg(vec + a.v_wc + c * odim + j), xc[c * RPX], y);
          if (a.act == WEKWS_ACT_SIGMOID) y = sigmoidf_acc(y);
          a.out[(size_t)(b0 + i * spt + s) * a.out_bstride + (size_t)tt * odim + j] = y;
        }
      }
    }
    __syncthreads();       // pass boundary
  }
}

}  // namespace

bool tcn_tc_eligible(const TcnTcArgs& a, int padmax) {
  if (a.idim % 8 != 0 || a.idim > 128 || a.odim > 8 || a.ktaps > 8 || a.ktaps < 2) return false;
  if (((padmax + 3) & ~3) + 8 > XCOLS) return false;
  return true;
}

// a chunk of T frames takes roundup4(padmax) + roundup4(T) columns of X per stream: long receptive fields leave room
// for fewer than 128 frames (XCOLS and the rounded pad are multiples of 4, so every chunk of this height fits)
int tcn_tc_max_T(int padmax) {
  const int room = XCOLS - ((padmax + 3) & ~3);
  return room < 128 ? room : 128;
}

int tcn_tc_launch(TcnTcArgs a, int padmax, cudaStream_t st) {
  WEKWS_REQUIRE(a.T >= 1 && a.T <= 128 && a.B >= 1, "tcn_tc_launch: bad shape");
  a.padr = (padmax + 3) & ~3;
  const int Lw = a.padr + ((a.T + 3) & ~3);
  a.spt = 128 / a.T;
  WEKWS_REQUIRE(a.spt >= 1 && Lw <= XCOLS, "tcn_tc_launch: tile does not fit");
  int smax = NTILE * a.spt;
  if (smax > XCOLS / Lw) smax = XCOLS / Lw;
  a.smax = smax;
  const int sms = device_sm_count();
  const int grid = a.B < sms ? a.B : sms;
  if (const int rc = opt_in_smem((const void*)tcn_tc_kernel, SMEM_TOTAL)) return rc;
  tcn_tc_kernel<<<grid, NT_TC, SMEM_TOTAL, st>>>(a);
  return check_launch("tcn_tc_kernel");
}

}  // namespace wekws
