// Dense Linear on the tensor cores (wgmma) for wide outputs: Y[rows][N] = act(X[rows][K] . W[N][K]^T + b), K <= 256,
// any N.  Used for the CTC classifier heads (classifier.py:63-67 with output_dim 2599, examples/hi_xiaowen/s0/conf/
// ds_tcn_ctc.yaml:31-42) behind the tensor-core DS-TCN backbone: at odim 2599 the classifier is 1.33 MFLOP per frame,
// 2.3x the whole backbone, and used to force the model onto the FP32 kernel.
//
// bf16 x3 operand split, fp32 accumulate (same arithmetic as the backbone kernels).  One CTA per 128-row tile
// (persistent over tiles):
//   * the tile's A operand (128 rows x K, hi | lo) is written to shared memory once per tile as K-major SWIZZLE_128B
//     images (global fp32 row -> split -> st.shared) and reused for every output tile;
//   * W streams from L2 as pre-swizzled K-major SWIZZLE_128B images (128 output columns x 64 K, hi | lo = 32 KB,
//     the format of dstcn_tc.cu) through a 2-slot cp.async.bulk ring;
//   * per output tile of 128 columns each of the two warpgroups runs K/64 slabs x 3 passes x 4 wgmma (M = 64, N = 128,
//     K = 16) into a register accumulator, then its epilogue (bias, activation, stores to global).
// Warps: 0-7 compute (two warpgroups of 64 rows), 8 weight loader.
#include "common.cuh"
#include "linear_tc.h"
#include "tc_common.cuh"

namespace wekws {
namespace {

using namespace tc;

constexpr int NCT = 256, NT = NCT + 32;
constexpr int W_SLOT = 32768, NW = 2;
constexpr int A_SLAB = 32768;                  // one 64-wide K slab of the tile's operand: hi (16 KB) then lo (16 KB)
constexpr int OFF_A = NW * W_SLOT;
constexpr int SMEM_BYTES = OFF_A + 4 * A_SLAB + 1024;
constexpr int NTILE = 128;     // output columns per accumulator

__device__ __forceinline__ void compute_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(NCT) : "memory"); }

__global__ void __launch_bounds__(NT, 1) linear_tc_kernel(const LinearTcArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
  __shared__ uint64_t w_bar[NW], w_free[NW];
  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);

  if (tid == 0) {
    for (int i = 0; i < NW; ++i) { mbar_init(&w_bar[i], 1); mbar_init(&w_free[i], NCT / 32); }
    mbar_fence_init();
  }
  __syncthreads();
  const int nslab = a.K / 64, ntn = (a.N + NTILE - 1) / NTILE;
  const int my_tiles = a.n_mtiles > (int)blockIdx.x ? (a.n_mtiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

  if (warp < NCT / 32) {
    // ================================================================== COMPUTE: operand rows, GEMMs, epilogues
    const int wg = warp >> 2, w = warp & 3, q4 = lane & 3;
    const uint32_t abase = smem_u32(base + OFF_A);
    uint32_t seq = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const long long tile0 = (long long)(blockIdx.x + it * gridDim.x) * 128;
      if (it > 0) compute_barrier();                 // every warpgroup's MMAs of the previous tile have read the operand
      {
        // thread (row, half): 8-value chunks c = half, half + 2, ... of the row -> hi / lo images
        const int row = tid & 127, half = tid >> 7;
        const long long r = tile0 + row;
        const bool live = r < a.rows;
        const float4* src = reinterpret_cast<const float4*>(a.x + r * a.x_stride);
        for (int c = half; c < a.K / 8; c += 2) {
          float v[8];
          const float4 f0 = live ? __ldg(src + 2 * c) : make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 f1 = live ? __ldg(src + 2 * c + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
          v[0] = f0.x; v[1] = f0.y; v[2] = f0.z; v[3] = f0.w; v[4] = f1.x; v[5] = f1.y; v[6] = f1.z; v[7] = f1.w;
          uint8_t* slab = base + OFF_A + (c >> 3) * A_SLAB;
          split_store8(v, slab, slab + 16384, sw128_offset(row, c & 7));
        }
      }
      fence_proxy_async();                           // generic-proxy stores -> visible to wgmma
      compute_barrier();
      const int rbase = 64 * wg + 16 * w + (lane >> 2);
      for (int n = 0; n < ntn; ++n) {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        for (int s = 0; s < nslab; ++s, ++seq) {
          const uint32_t slot = seq % NW;
          mbar_wait(&w_bar[slot], (seq / NW) & 1);
          const uint64_t whi = make_sdesc_sw128(smem_u32(base + slot * W_SLOT)), wlo = whi + (16384 >> 4);
          const uint64_t ahi = make_sdesc_sw128(abase + s * A_SLAB + wg * 8192), alo = ahi + (16384 >> 4);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(acc, ahi + 2 * k, whi + 2 * k, (s == 0 && k == 0) ? 0u : 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(acc, alo + 2 * k, whi + 2 * k, 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(acc, ahi + 2 * k, wlo + 2 * k, 1u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_reg_fence(acc);
          __syncwarp();
          if (lane == 0) mbar_arrive(&w_free[slot]);
        }
        const int n0 = n * NTILE;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const long long r = tile0 + rbase + 8 * h;
          if (r >= a.rows) continue;
          float* orow = a.out + r * a.out_stride;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int c0 = n0 + 8 * j + 2 * q4;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              if (c0 + e < a.N) {
                float y = acc[4 * j + 2 * h + e] + __ldg(a.bias + c0 + e);
                if (a.act == WEKWS_ACT_SIGMOID) y = sigmoidf_acc(y);
                orow[c0 + e] = y;
              }
            }
          }
        }
      }
    }
  } else {
    // ================================================================== WEIGHT LOADER (lane 0): images [n tile][slab]
    if (lane == 0) {
      const uint32_t total = (uint32_t)my_tiles * (uint32_t)ntn * (uint32_t)nslab, per = (uint32_t)ntn * (uint32_t)nslab;
      for (uint32_t seq = 0; seq < total; ++seq) {
        const uint32_t slot = seq % NW;
        if (seq >= NW) mbar_wait_backoff(&w_free[slot], ((seq / NW) - 1) & 1);
        mbar_arrive_expect_tx(&w_bar[slot], W_SLOT);
        bulk_g2s(base + slot * W_SLOT, a.wimg + (size_t)(seq % per) * W_SLOT, W_SLOT, &w_bar[slot]);
      }
    }
  }
}

}  // namespace

size_t linear_tc_image_bytes(int N, int K) { return (size_t)((N + NTILE - 1) / NTILE) * (size_t)(K / 64) * W_SLOT; }
bool linear_tc_eligible(int N, int K) { return K >= 64 && K <= 256 && K % 64 == 0 && N >= 1; }

void linear_tc_pack(uint8_t* dst, const float* wt, int ldn, int N, int K) {
  const int ntn = (N + NTILE - 1) / NTILE, nslab = K / 64;
  for (int nt = 0; nt < ntn; ++nt)
    for (int s = 0; s < nslab; ++s)
      tc::write_sw128_bf16x3(dst + (size_t)(nt * nslab + s) * W_SLOT, NTILE, wt + (size_t)64 * s * ldn + nt * NTILE, 1,
                             ldn, N - nt * NTILE, 64);
}

int linear_tc_launch(LinearTcArgs a, cudaStream_t st) {
  WEKWS_REQUIRE(a.rows >= 1 && linear_tc_eligible(a.N, a.K), "linear_tc_launch: unsupported shape (rows %lld, N %d, K %d)",
                (long long)a.rows, a.N, a.K);
  WEKWS_REQUIRE(((uintptr_t)a.x & 15) == 0 && (a.x_stride & 3) == 0, "linear_tc_launch: input rows must be 16-byte aligned");
  a.n_mtiles = (int)((a.rows + 127) / 128);
  if (const int rc = opt_in_smem((const void*)linear_tc_kernel, SMEM_BYTES)) return rc;
  const int sms = device_sm_count();
  const int grid = a.n_mtiles < sms ? a.n_mtiles : sms;
  linear_tc_kernel<<<grid, NT, SMEM_BYTES, st>>>(a);
  return check_launch("linear_tc_kernel");
}

}  // namespace wekws
