// Tensor-core (wgmma) fused forward for the depthwise-separable TCN backbone with hidden_dim 256
// (reference wekws/model/tcn.py:91-119 DsCnnBlock inside TCN :122-166, ds_tcn.yaml; BatchNorm folded):
//     per block:  a = ReLU(dw_k8,dil(cat(cache, x)))   o = ReLU(W_pw . a + b)   x' = o + x
// The pointwise 256x256 GEMM carries 97 % of the FLOPs and runs on wgmma with the bf16x3 split; the
// depthwise taps, BN/ReLU/residual and the classifier stay in FP32 on the CUDA cores.
//
// One CTA per SM owns a tile of up to 120 frames (spt = 120 / T whole streams) for the whole network:
//   * X[256][120] fp32, the residual stream (frames only), lives in shared memory (120 KB);
//   * the cache (halo) columns of a block are NOT staged: 256 channels x 56 columns x 3 streams would not fit
//     next to X, so the depthwise taps that reach back before the chunk read the cache straight from
//     global memory (lanes = consecutive frames, so a warp reads contiguous floats of one cache row);
//   * the depthwise output is produced 64 channels (one K slab) at a time, split into bf16 hi/lo and written to a
//     K-major SWIZZLE_128B operand image in shared memory;
//   * the accumulator D[128][256] fp32 lives in registers: warpgroup g holds output channels [64 g, 64 g + 64) of all
//     128 rows (two m64n64 accumulators); every slab issues 3 x 4 x 2 wgmma per warpgroup whose B operand is a
//     pre-swizzled 32 KB weight image (128 output channels x 64 K, hi | lo) streamed from L2 through a 2-slot ring by
//     cp.async.bulk (the 256 KB of a block's weights do not fit);
//   * depthwise coefficients of the current block (9 KB) are staged by one bulk copy per block.
// Warp roles: 16 compute warps (row = 32 * (warp % 4) + lane, channel group = warp / 4; warpgroup = warp / 4) + 1 weight
// loader warp.
#include <type_traits>

#include "common.cuh"
#include "dstcn_tc.h"
#include "tc_common.cuh"

namespace wekws {

namespace {

using namespace tc;

constexpr int NCW = 16, NCT = NCW * 32, NT_TC = NCT + 32;
constexpr int C = 256, KT = 8;
constexpr int RPX = 120;                                   // frames per tile == row pitch of X
constexpr int X_BYTES = C * RPX * 4;                       // 122880
constexpr int W_SLOT = 32768, NW = 2;                      // the two output halves of one K slab
constexpr int A_BYTES = 32768;                             // operand image of one K slab: hi [128][64] then lo
constexpr int COEF_FLOATS = (KT + 1) * C;                  // [tap][channel] then folded bias
constexpr int OFF_W = 0, OFF_A = NW * W_SLOT, OFF_X = OFF_A + A_BYTES, OFF_COEF = OFF_X + X_BYTES;
constexpr int SMEM_TOTAL = OFF_COEF + COEF_FLOATS * 4 + 1024;   // 231424
static_assert(SMEM_TOTAL <= 232448, "exceeds the 227 KB of shared memory a CTA may use");

__device__ __forceinline__ void compute_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(NCT) : "memory"); }
__device__ __forceinline__ float ld_global_f32(const float* p) {
  float v;
  asm("ld.global.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
// predicated global load: 0 when pred == 0 (the address is then not dereferenced)
__device__ __forceinline__ float ld_global_f32_pred(const float* p, uint32_t pred) {
  float v;
  asm volatile(
      "{\n\t"
      ".reg .pred q;\n\t"
      "setp.ne.b32 q, %2, 0;\n\t"
      "mov.f32 %0, 0f00000000;\n\t"
      "@q ld.global.f32 %0, [%1];\n\t"
      "}"
      : "=f"(v)
      : "l"(p), "r"(pred));
  return v;
}

// PP: compile-time cache row pitch (floats) so the cache loads get immediate offsets; 0 = read it from the arguments
template <int PP>
__global__ void __launch_bounds__(NT_TC, 1) dstcn_tc_kernel(const DsTcArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
  __shared__ uint64_t coef_bar, w_bar[NW], w_free[NW];
  __shared__ int store_ctr[1];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const bool is_loader = warp == NCW;
  const int q = warp & 3, g = (warp >> 2) & 3;
  const int row = 32 * q + lane;
  const int T = a.T, P = PP ? PP : a.P;
  const float* vec = a.vec;
  float* X = reinterpret_cast<float*>(base + OFF_X);
  float* coef = reinterpret_cast<float*>(base + OFF_COEF);
  uint8_t* Wring = base + OFF_W;
  uint8_t* Aimg = base + OFF_A;

  if (tid == 0) {
    mbar_init(&coef_bar, 1);
    for (int i = 0; i < NW; ++i) { mbar_init(&w_bar[i], 1); mbar_init(&w_free[i], 8); }
    mbar_fence_init();
  }
  __syncthreads();
  uint32_t coef_par = 0;
  const int natoms = (a.idim + 63) / 64;
  const int spt = a.spt;
  const int nlin = 2 * natoms;
  const int nitems = nlin + a.nblocks * 8;          // weight images per pass

  const int sb = (int)(((long long)a.B * blockIdx.x) / gridDim.x);
  const int se = (int)(((long long)a.B * (blockIdx.x + 1)) / gridDim.x);
  int done = sb;
  uint32_t gu = 0;                                   // compute: weight images consumed so far (in pairs)

  auto load_coef = [&](int blk) {                    // one thread
    fence_proxy_async();                             // the area was read/written through the generic proxy
    mbar_arrive_expect_tx(&coef_bar, COEF_FLOATS * 4);
    bulk_g2s(coef, vec + a.v_blocks + (size_t)blk * a.v_blk_stride, COEF_FLOATS * 4, &coef_bar);
  };
  uint32_t gl = 0;                                   // loader: weight images issued so far

  while (done < se) {
    const int remaining = se - done;
    const int passes_left = (remaining + spt - 1) / spt;
    const int ns = (remaining + passes_left - 1) / passes_left;
    const int b0 = done;
    done += ns;
    const int rows = ns * T;

    if (is_loader) {
      // ================================================================== WEIGHT LOADER (lane 0): the pass's images
      if (lane == 0) {
        for (int n = 0; n < nitems; ++n, ++gl) {
          const uint32_t slot = gl % NW;
          if (gl >= NW) mbar_wait_backoff(&w_free[slot], ((gl / NW) - 1) & 1);
          mbar_arrive_expect_tx(&w_bar[slot], W_SLOT);
          bulk_g2s(Wring + slot * W_SLOT, a.wimg + (size_t)n * W_SLOT, W_SLOT, &w_bar[slot]);
        }
      }
    } else {
      // ================================================================== COMPUTE WARPS
      // Rows are ordered frame-major: row = t * ns + s, and X[c][row] likewise, so a tap is a column shift of
      // j * d * ns and the rows of a warp span ~32 / ns consecutive frames: only the warps holding the first frames
      // of the chunk reach back into the cache, and only for their first taps.
      const bool valid = row < rows, q_live = 32 * q < rows;
      const int t = valid ? row / ns : 0, s = valid ? row - t * ns : 0;
      const int t_min = (32 * q) / ns;                 // first frame of this warp's rows
      const int q4 = lane & 3, rb = 16 * q + (lane >> 2);   // wgmma fragment: rows rb + 8 h (+ 64 mt) of warpgroup g
      const uint32_t abase = smem_u32(Aimg);
      if (tid == 0) load_coef(0);
      float acc[2][32];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[mt][i] = 0.f;
      // the slab's operand image is complete: every warpgroup adds A * W^T for its 64 output channels (image half g / 2
      // of the current pair, rows 64 (g % 2) of it); once the MMAs are done the image and the weight slot are free
      auto gemm_slab = [&](int ksteps, bool fresh) {
        fence_proxy_async();
        compute_barrier();
        const uint32_t slot = (uint32_t)(g >> 1);
        mbar_wait(&w_bar[slot], (gu / NW) & 1);
        const uint64_t dwh = make_sdesc_sw128(smem_u32(Wring + slot * W_SLOT) + (uint32_t)(g & 1) * 8192u), dwl = dwh + (16384 >> 4);
        wgmma_fence();
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          const uint64_t ahi = make_sdesc_sw128(abase + mt * 8192), alo = ahi + (16384 >> 4);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_ss(acc[mt], ahi + 2 * k, dwh + 2 * k, (fresh && k == 0) ? 0u : 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_ss(acc[mt], alo + 2 * k, dwh + 2 * k, 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_ss(acc[mt], ahi + 2 * k, dwl + 2 * k, 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(acc[0]);
        wgmma_reg_fence(acc[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&w_free[slot]);
        gu += NW;
        compute_barrier();                             // the operand image may be rewritten
      };
      // byte offset of 8-value chunk `ch` (0..7) of this thread's row in the operand image (hi; lo at + 16384)
      const uint32_t arow = (uint32_t)row * 128u;
      auto a_off = [&](int ch) { return arow + (uint32_t)((ch ^ (row & 7)) << 4); };

      // ---- features (+CMVN) -> bf16 hi/lo operand of the first Linear, one 64-wide K slab at a time
      for (int at = 0; at < natoms; ++at) {
        const int nch = min(8, ((a.idim - 64 * at + 15) >> 4) * 2);
        const float* src0 = a.feats + (size_t)(b0 + s) * a.feat_bstride + (size_t)t * a.idim + 64 * at;
        for (int ch = g; ch < nch; ch += 4) {
          float v[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) v[u] = 0.f;
          const int k0 = 64 * at + ch * 8;
          if (valid && k0 < a.idim) {
            const float4 f0 = __ldg(reinterpret_cast<const float4*>(src0 + ch * 8));
            const float4 f1 = __ldg(reinterpret_cast<const float4*>(src0 + ch * 8) + 1);
            v[0] = f0.x; v[1] = f0.y; v[2] = f0.z; v[3] = f0.w; v[4] = f1.x; v[5] = f1.y; v[6] = f1.z; v[7] = f1.w;
            if (a.has_cmvn) {
#pragma unroll
              for (int u = 0; u < 8; ++u) v[u] = (v[u] - __ldg(vec + a.v_mean + k0 + u)) * __ldg(vec + a.v_istd + k0 + u);
            }
          }
          split_store8(v, Aimg, Aimg + 16384, a_off(ch));
        }
        const int rem = a.idim - 64 * at;
        gemm_slab(rem >= 64 ? 4 : (rem + 15) >> 4, at == 0);
      }
      // ---- x = relu(D + bp) -> X
      auto epilogue = [&](const float* bias, bool residual) {
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = 64 * mt + rb + 8 * h;
            if (r >= rows) continue;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int c = 64 * g + 8 * j + 2 * q4;
              const float2 bv = __ldg(reinterpret_cast<const float2*>(bias + c));
              float* xp = X + c * RPX + r;
              const float o0 = fmaxf(acc[mt][4 * j + 2 * h] + bv.x, 0.f), o1 = fmaxf(acc[mt][4 * j + 2 * h + 1] + bv.y, 0.f);
              xp[0] = residual ? o0 + xp[0] : o0;
              xp[RPX] = residual ? o1 + xp[RPX] : o1;
            }
          }
      };
      epilogue(vec + a.v_bp, false);
      if (tid == 0) store_ctr[0] = 0;
      compute_barrier();

      for (int blk = 0; blk < a.nblocks; ++blk) {
        const int d = a.dil[blk], pad = d * (KT - 1), off = a.coff[blk];
        mbar_wait(&coef_bar, coef_par);
        coef_par ^= 1u;
        // taps that reach back before the chunk read cat index < pad from the cache row of this stream
        const float* crow = valid && a.in_cache != nullptr ? a.in_cache + (size_t)(b0 + s) * C * P + off : nullptr;
        const int t0 = valid ? t : -(1 << 20);         // padding rows: every cache-capable tap takes the absent-cache path
        // taps j < jc can need the cache for some row of this warp (t_min + j d < pad); rounded up to a compiled variant
        const int jc = pad > t_min ? min(KT - 1, (pad - t_min + d - 1) / d) : 0;

        // depthwise taps of 8 channels -> ReLU -> bf16 hi/lo -> the operand image.  Taps j < JC are compiled with
        // a predicated global load (cache part) next to the shared load (frame part), the rest with the shared load
        // only; everything is branch-free so the loads of a chunk are in flight together.
        auto dw_chunk = [&](auto jct, int c0, int ach) {
          constexpr int JC = decltype(jct)::value;
          float acc[8];
          {
            const float4 b0v = *reinterpret_cast<const float4*>(coef + KT * C + c0);
            const float4 b1v = *reinterpret_cast<const float4*>(coef + KT * C + c0 + 4);
            acc[0] = b0v.x; acc[1] = b0v.y; acc[2] = b0v.z; acc[3] = b0v.w;
            acc[4] = b1v.x; acc[5] = b1v.y; acc[6] = b1v.z; acc[7] = b1v.w;
          }
          const float* xc = X + c0 * RPX + row;
          const float* gc = crow + (size_t)c0 * P + t0;
#pragma unroll
          for (int j = 0; j < KT; ++j) {
            const float4 w0 = *reinterpret_cast<const float4*>(coef + j * C + c0);
            const float4 w1 = *reinterpret_cast<const float4*>(coef + j * C + c0 + 4);
            const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
            const int sh = (j * d - pad) * ns;         // column shift of the frame part
            float v[8];
            if (j < JC) {
              const bool in_c = t0 + j * d < pad, pg = in_c && crow != nullptr;
              const float* xp = in_c ? X + c0 * RPX : xc + sh;
              const float* gp = gc + j * d;
#pragma unroll
              for (int u = 0; u < 8; ++u) {
                const float vx = xp[u * RPX];
                const float vg = pg ? ld_global_f32(gp + u * P) : 0.f;   // L1-cached: neighbouring taps/rows re-read it
                v[u] = in_c ? vg : vx;
              }
            } else {
#pragma unroll
              for (int u = 0; u < 8; ++u) v[u] = xc[sh + u * RPX];
            }
#pragma unroll
            for (int u = 0; u < 8; ++u) acc[u] = fmaf(w[u], v[u], acc[u]);
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) acc[u] = fmaxf(acc[u], 0.f);
          split_store8(acc, Aimg, Aimg + 16384, a_off(ach));
        };

        for (int ks = 0; ks < 4; ++ks) {
          if (q_live) {
#pragma unroll 1
            for (int half = 0; half < 2; ++half) {
              const int c0 = 64 * ks + 16 * g + 8 * half, ach = 2 * g + half;
              if (jc == 0) dw_chunk(std::integral_constant<int, 0>{}, c0, ach);
              else if (jc <= 3) dw_chunk(std::integral_constant<int, 3>{}, c0, ach);
              else if (jc <= 5) dw_chunk(std::integral_constant<int, 5>{}, c0, ach);
              else dw_chunk(std::integral_constant<int, 7>{}, c0, ach);
            }
          }
          if (ks == 3) {
            // New cache slices (tcn.py:54: last `pad` columns of cat(cache, x)), stored before the last slab's GEMM
            // so the epilogue (which overwrites x) cannot start before every store has been issued.  x is
            // stable during the whole depthwise phase, so a warp starts as soon as its own taps are done and takes
            // row groups from a shared counter: the warps without cache taps finish early and do most of the moving.
            // Only when out_cache aliases in_cache must every warp first be past its last read of the old slices.
            if (a.aliased) compute_barrier();
            const int L = pad <= 8 ? 8 : pad <= 16 ? 16 : 32, npr = 32 / L, sub = lane / L, pl = lane - sub * L;
            const int ngroups = ns * C / npr;          // a group = npr rows of `pad` floats, one warp iteration per L floats
            const size_t pbase = (size_t)b0 * C * P + off;
            const float* ic = a.in_cache != nullptr ? a.in_cache + pbase : nullptr;
            float* oc = a.out_cache + pbase;
            const int from_cache = pad - T;            // elements p < pad - T come from the old slice (column p + T)
            for (;;) {
              int g0 = 0;
              if (lane == 0) g0 = atomicAdd(store_ctr, 4);
              g0 = __shfl_sync(0xffffffffu, g0, 0);
              if (g0 >= ngroups) break;
              const int g1 = min(g0 + 4, ngroups);
              for (int gi = g0; gi < g1; ++gi) {
                const int r = gi * npr + sub, ss = r >> 8, c = r & (C - 1), rp = r * P;
                const float* xrow = X + c * RPX + ss + (T - pad) * ns;      // element p of the new slice = xrow[p * ns]
                for (int p0 = 0; p0 < pad; p0 += L) {  // ascending: a row shifts left by T, reads stay ahead of writes
                  const int p = p0 + pl;
                  const bool act = p < pad, fx = p >= from_cache;
                  const float xv = xrow[(act && fx ? p : pad - T) * ns];
                  float v = 0.f;
                  if (act && !fx && ic != nullptr) v = __ldcg(ic + rp + T + p);
                  v = fx ? xv : v;
                  if (a.aliased) __syncwarp();
                  if (act) oc[rp + p] = v;
                }
              }
            }
          }
          gemm_slab(4, ks == 0);
          if (ks == 3 && tid == 0 && blk + 1 < a.nblocks) load_coef(blk + 1);   // every warp is past this block's taps
        }
        // ---- x' = relu(D + b_pw) + x -> X                                   (tcn.py:60: no ReLU after the add)
        epilogue(vec + a.v_blocks + blk * a.v_blk_stride + (KT + 1) * C, true);
        if (tid == 0) store_ctr[0] = 0;
        compute_barrier();
      }

      // ---- classifier + activation on x (tcn.py:165 -> classifier.py:63-67); partial sums reuse the coefficient area
      const int odim = a.odim;
      if (a.hidden != nullptr) {
        // wide classifier heads run as their own tensor-core GEMM (linear_tc.cu): hand over x as (stream, frame, 256) rows.
        // lanes = consecutive rows (conflict-free reads of X[c][row]); each warp walks the channels
        for (int c = warp; c < C; c += NCW) {
          for (int r = lane; r < rows; r += 32) {
            const int tt = r / ns, ss = r - tt * ns;
            a.hidden[(size_t)(b0 + ss) * a.hidden_bstride + (size_t)tt * C + c] = X[c * RPX + r];
          }
        }
      } else {
      {
        const int r = tid & 127, part = tid >> 7;
        if (r < rows) {
          for (int j = 0; j < odim; ++j) {
            float y = 0.f;
#pragma unroll 8
            for (int c = 64 * part; c < 64 * part + 64; ++c) y = fmaf(__ldg(vec + a.v_wc + c * odim + j), X[c * RPX + r], y);
            coef[(j * 4 + part) * 128 + r] = y;
          }
        }
      }
      compute_barrier();
      for (int idx = tid; idx < rows * odim; idx += NCT) {
        const int r = idx / odim, j = idx - r * odim;
        float y = __ldg(vec + a.v_bc + j) + coef[(j * 4 + 0) * 128 + r] + coef[(j * 4 + 1) * 128 + r] +
                  coef[(j * 4 + 2) * 128 + r] + coef[(j * 4 + 3) * 128 + r];
        if (a.act == WEKWS_ACT_SIGMOID) y = sigmoidf_acc(y);
        const int tt = r / ns, ss = r - tt * ns;
        a.out[(size_t)(b0 + ss) * a.out_bstride + (size_t)tt * odim + j] = y;
      }
    }
      }
    __syncthreads();       // pass boundary
  }
}

}  // namespace

bool dstcn_tc_eligible(const DsTcArgs& a, int hdim, bool cls_gemm) {
  return hdim == C && a.ktaps == KT && a.idim % 8 == 0 && a.idim >= 8 && a.idim <= 128 && a.odim >= 1 && (a.odim <= 4 || cls_gemm) &&
         a.v_blocks % 4 == 0 && a.v_blk_stride % 4 == 0;
}

int dstcn_tc_max_T() { return RPX; }

int dstcn_tc_launch(DsTcArgs a, cudaStream_t st) {
  WEKWS_REQUIRE(a.T >= 1 && a.T <= RPX && a.B >= 1, "dstcn_tc_launch: bad shape");
  a.spt = RPX / a.T;
  {
    const size_t bytes = (size_t)a.B * C * a.P * sizeof(float);
    const char* i0 = reinterpret_cast<const char*>(a.in_cache);
    const char* o0 = reinterpret_cast<const char*>(a.out_cache);
    a.aliased = a.in_cache != nullptr && i0 < o0 + bytes && o0 < i0 + bytes;
  }
  const int sms = device_sm_count();
  const int tiles = (a.B + a.spt - 1) / a.spt;
  const int grid = tiles < sms ? tiles : sms;
  auto* kernel = a.P == 105 ? dstcn_tc_kernel<105> : dstcn_tc_kernel<0>;   // ds_tcn.yaml: k = 8, dilations 1, 2, 4, 8
  if (const int rc = opt_in_smem((const void*)kernel, SMEM_TOTAL)) return rc;
  kernel<<<grid, NT_TC, SMEM_TOTAL, st>>>(a);
  return check_launch("dstcn_tc_kernel");
}

}  // namespace wekws
