// Tensor-core (wgmma) fused MDTC forward for hidden_dim 64 -- the throughput path.
//
// Same math as conv_backbone.cu (KWSModel.forward, reference wekws/model/kws_model.py:65-76 with
// mdtc.py:95-121 blocks, BatchNorm folded), but every dense GEMM (first Linear 80->64 and the 34
// pointwise 64x64 convolutions) runs on the tensor cores:
//   * bf16 "x3" operand split (tc_common.cuh): result within ~2^-16 of fp32 (posterior error ~1e-5, bar 1e-4);
//   * the A operand (activations) never leaves the registers: the depthwise conv and the pointwise-1 epilogue
//     produce it directly in the wgmma A-fragment layout, and the pointwise-1 accumulator IS the A fragment of the
//     pointwise-2 GEMM; B (weights) is a pre-swizzled K-major SWIZZLE_128B image in shared memory, streamed by
//     cp.async.bulk into a 2-slot ring;
//   * a 128-row tile is one GROUP of two warpgroups (64 rows each, accumulator 64 x 64 fp32 in registers), and the
//     groups run the network independently of each other (a named barrier per group over its live warps), so the
//     CUDA-core phases of one tile overlap the tensor-core phases of the other; a warpgroup with no row in the pass
//     only keeps the weight ring and the loader's barriers in step.
//
// One CTA per SM holds ALL of its streams (up to 7 x 40 frames) resident for the whole network.  The residual stream is
// CHANNEL-MINOR: X[col][64 ch] (272 B per frame column: 256 B of channels and one 16-byte pad chunk that staggers the
// banks; every stream's cache slice in the columns directly in front of its frames, so a dilated tap is a column offset).
//
// 20 warps = 5 warpgroups: 16 compute (2 groups x 2 warpgroups), then the service warpgroup: 1 weight ring warp,
// 2 loaders (cache slices by 2-D TMA tensor copies into landing slots, transposed into X) and one warp that only keeps
// the warpgroup whole.  The CTA launches at 96 registers per thread; after the prologue the service warpgroup gives
// all but 40 of its registers to the compute warpgroups (setmaxnreg), which then hold 104.
#include <stdlib.h>

#include "common.cuh"
#include "mdtc_tc.h"
#include "tc_common.cuh"

// per-phase cycle counters of the loaders and of one compute warp per group (debug builds with -DMDTC_TIMING=1 only)
#ifndef MDTC_TIMING
#define MDTC_TIMING 0
#endif
#if MDTC_TIMING
#define TPH(acc) { const long long t_now_ = clock64(); acc += t_now_ - t_last_; t_last_ = t_now_; }
#else
#define TPH(acc)
#endif

namespace wekws {

namespace {

using namespace tc;

constexpr int NG = 2;                      // row tiles in flight == compute groups
constexpr int WPG = 8;                     // warps per group (tile): two warpgroups of 64 rows each
constexpr int NCW = NG * WPG;              // compute warps (16)
constexpr int W_WGT = NCW;                 // warp 16: weight ring
constexpr int W_LD = W_WGT + 1;            // warps 17..18: cache loaders, one per tile
constexpr int NT_TC = (NCW + 4) * 32;      // 640 threads: five whole warpgroups, launched at 96 registers per thread
constexpr int REG_SERVICE = 40;            // registers per thread after the handoff: service warpgroup ...
constexpr int REG_COMPUTE = 104;           // ... and compute warpgroups (4 x 104 + 40 <= 5 x 96)
static_assert(W_LD + NG <= NCW + 4, "the service roles must fit in the service warpgroup");
static_assert(4 * REG_COMPUTE + REG_SERVICE <= 5 * 96, "the handoff must not take more registers than the CTA holds");
constexpr int C = 64;
constexpr int XCOLS = 504;                 // frame columns of X (n_streams * Lw <= XCOLS)
constexpr int X_COL = 272;                 // bytes per frame column of X: 64 fp32 + one 16-byte pad chunk
constexpr int X_BYTES = XCOLS * X_COL;     // 137088
constexpr int STG_FLOATS = 64 * 32;        // TMA landing slot: one stream's cache slice [64][pad <= 32]
constexpr int NSLOT = 7;                   // TMA landing slots, shared out among the tiles' loaders by stream count
constexpr int NSLOT_HEAD = 6;              // the head variant gives one slot's room to its pool
constexpr int W_SLOT = 16384;              // hi + lo image of one 64x64 matrix
constexpr int OFF_W = 0;                                   // 1024-aligned: SWIZZLE_128B images
constexpr int OFF_X = OFF_W + 2 * W_SLOT;                  // 32768
constexpr int OFF_STG = OFF_X + X_BYTES;                   // 169856 (128-aligned: TMA destination)
constexpr int OFF_WC = OFF_STG + NSLOT * STG_FLOATS * 4;            // per-frame classifier weights [64][odim <= 8]
constexpr int SMEM_TOTAL = OFF_WC + C * 8 * 4 + 1024;                // 230272, incl. alignment slack
constexpr int POOL_SPT = 16;                               // streams per tile at the shortest chunk (T = 8)
constexpr int OFF_POOL = OFF_STG + NSLOT_HEAD * STG_FLOATS * 4;       // head variant: pooled sums [NG][POOL_SPT][64]
constexpr int SMEM_TOTAL_HEAD = OFF_POOL + NG * POOL_SPT * C * 4 + 1024;   // 228224
static_assert(OFF_W % 1024 == 0 && OFF_X % 128 == 0 && OFF_STG % 128 == 0, "misaligned shared-memory region");
static_assert(SMEM_TOTAL <= 232448, "exceeds the 227 KB of shared memory a CTA may use");
static_assert(SMEM_TOTAL_HEAD <= 232448, "exceeds the 227 KB of shared memory a CTA may use");

// named barrier of tile grp's nlw live compute warps
__device__ __forceinline__ void group_barrier(int grp, int nlw) {
  asm volatile("bar.sync %0, %1;" ::"r"(grp + 1), "r"(32 * nlw) : "memory");
}
__device__ __forceinline__ float2 lds_f2(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_f2(uint32_t addr, float x, float y) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(x), "f"(y) : "memory");
}
// Layout of X: frame column col holds its 64 channels in the first 256 of its X_COL = 272 bytes; the 16-byte chunk with
// channels 8m..8m+3 sits at byte 16 m, channels 8m+4..8m+7 at 128 + 16 m:
//   address(col, 8m + 4h + u) = xs + 272 col + 16 m + 128 h + 4 u
// Chunk m of column col falls in bank group (col + m) mod 8, so for a fixed m the columns spread over the banks as they
// would under an XOR swizzle (tests/test_mdtc_x_layout.py counts every access pattern), while the chunk offset 16 m
// stays an immediate of the load: x_addr(xs, col, 8 m + r) == x_addr(xs, col, r) + 16 m for r < 8.
__device__ __forceinline__ uint32_t x_addr(uint32_t xs, int col, int ch) {
  return xs + (uint32_t)col * X_COL + 16u * (uint32_t)(ch >> 3) + 128u * (uint32_t)((ch >> 2) & 1) + 4u * (uint32_t)(ch & 3);
}
// 2-D TMA tensor copy global -> shared (box given by the tensor map), completion on an mbarrier
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, int c0, int c1, uint64_t* bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(c0), "r"(c1), "r"(smem_u32(bar))
               : "memory");
}


// The service roles run in the service warpgroup's own pass loop, after its setmaxnreg.dec.  They are inlined there:
// as __noinline__ functions the call ABI pinned registers, and at 40 registers the loader spilled 128-136 bytes.
// Inlined, with its transpose loops kept rolled, it fits (KT = 5) or keeps 1-3 spill instructions (KT = 0).
// (Under the wgmma fragment layout the per-block tap / bias constants are read with lane-indexed LDC from the parameter bank, four distinct addresses per warp.  Reading them instead from a
// fragment-ordered global array with __ldg was measured 11 % slower on H100: see DESIGN.md section 3.)
struct Bars {
  uint64_t *halo_bar, *h_free, *w_bar, *w_free, *stg_bar;
};

// WEIGHT RING (one thread): slot 0 carries Linear atom 0, W1(0), W1(1), ...; slot 1 [Linear atom 1], W2(0), ...
__device__ __forceinline__ void weights_role(const TcArgs& a, uint8_t* base, Bars B, int K, int natoms, uint32_t& wf_par,
                                             bool first_pass) {
  uint8_t* Wslot[2] = {base + OFF_W, base + OFF_W + W_SLOT};
  auto load_w = [&](int slot, const uint8_t* src) {
    mbar_arrive_expect_tx(&B.w_bar[slot], W_SLOT);
    bulk_g2s(Wslot[slot], src, W_SLOT, &B.w_bar[slot]);
  };
  auto wait_free = [&](int slot) {             // every tile's MMAs on the slot's current weights are done
    mbar_wait_backoff(&B.w_free[slot], (wf_par >> slot) & 1);
    wf_par ^= 1u << slot;
  };
  load_w(0, a.wimg);
  if (natoms > 1) load_w(1, a.wimg + W_SLOT);
  for (int b = 0; b <= a.nblocks; ++b) {
    const uint8_t* wb = a.wimg + (size_t)(2 + 2 * b) * W_SLOT;
    wait_free(0);
    if (b < a.nblocks) load_w(0, wb);
    if (b > 0 || natoms > 1) wait_free(1);
    if (b < a.nblocks) load_w(1, wb + W_SLOT);
  }
}

// LOADER WARP i serves tile i only: per (block, stream of the tile) one 2-D TMA copy [64][pad] into a landing slot,
// then the warp transposes it into the pad columns in front of the stream's frames in X.  A dedicated loader per tile
// means a group never queues behind another tile's slices (the round-2 profile showed the groups waiting 14 % of the
// time on halo_bar with two loaders walking the tiles in order).  The tile's ring of `nsl` landing slots is refilled
// the moment a slot is drained, i.e. the copy for the same stream of the NEXT block is in flight a whole block ahead.
__device__ __forceinline__ void loader_role(const TcArgs& a, uint8_t* base, Bars B, int i, int lane, int K, int ns,
                                            int b0, int ntile, int nslot, uint32_t& hf_par) {
  if (i >= ntile) return;
  float* STG = reinterpret_cast<float*>(base + OFF_STG);
  const uint32_t xs = smem_u32(base) + OFF_X;
  const int T = a.T, PADR = a.padr, Lw = a.padr + T, spt = a.spt;
  const int nst = min(spt, ns - i * spt), sg0 = i * spt;          // my streams: sg0 .. sg0 + nst
  const int njobs = a.nblocks * nst;
  const bool have_cache = a.in_cache != nullptr;
  // landing slots of tile t: the streams' share of the nslot slots (each tile at least one; ns <= nslot: one per stream)
  int slot0 = 0, nsl = 1;
  {
    int used = 0;
    for (int t = 0; t < ntile; ++t) {
      const int n_t = min(spt, ns - t * spt);
      int want = ns <= nslot ? n_t : max(1, (nslot * n_t) / ns);
      const int left = nslot - used - (ntile - 1 - t);               // keep one slot for every later tile
      if (want > left) want = left;
      if (t == i) { slot0 = used; nsl = want; }
      used += want;
    }
  }
  auto issue_tma = [&](int k) {                    // lane 0; job k = (blk, my m-th stream)
    const int blk = k / nst, sg = sg0 + (k - blk * nst);
    const int pad = a.dil[blk] * (K - 1);
    const uint32_t slot = slot0 + (uint32_t)k % nsl;
    mbar_arrive_expect_tx(&B.stg_bar[slot], (uint32_t)(C * pad * 4));
    tma_load_2d(STG + slot * STG_FLOATS, &a.tmap[a.tmap_idx[blk]], a.coff[blk], (b0 + sg) * C, &B.stg_bar[slot]);
  };
  // (an up-front cp.async.bulk.prefetch.L2 of the streams' whole cache rows was measured: 3 % slower)
  if (have_cache && lane == 0)
    for (int k0 = 0; k0 < nsl && k0 < njobs; ++k0) issue_tma(k0);
  int k = 0;
#if MDTC_TIMING
  long long t_hf = 0, t_stg = 0, t_tr = 0;
  long long t_last_ = clock64();
#endif
  for (int blk = 0; blk < a.nblocks; ++blk) {
    const int pad = a.dil[blk] * (K - 1);
    // X's pad columns of the tile are free once the depthwise conv of blk-1 is done (at blk 0: from the start)
    if (blk > 0) {
      if (lane == 0) mbar_wait_backoff(&B.h_free[i], hf_par & 1);
      hf_par ^= 1u;
      __syncwarp();
    }
    TPH(t_hf)
    // one 4-channel x 4-column item: four LDS.128 along the slot's (time-minor) channel rows, a register transpose,
    // four STS.128 (4 channels of one column each) -- 8 shared-memory instructions per 64 bytes
    const int lgg = 31 - __clz(pad >> 2);          // column groups of 4 per channel row (pad is a power of two >= 4)
    auto move_item = [&](const float* slotp, int colb, int r) {
      const int cq = r >> lgg, jg = r & ((1 << lgg) - 1);
      const float4* s4 = reinterpret_cast<const float4*>(slotp + 4 * cq * pad + 4 * jg);
      const float4 r0 = s4[0], r1 = s4[pad >> 2], r2 = s4[2 * (pad >> 2)], r3 = s4[3 * (pad >> 2)];
      const uint32_t d = x_addr(xs, colb + 4 * jg, 4 * cq);
      sts_2x2(d, pack2(r0.x, r1.x), pack2(r2.x, r3.x));
      sts_2x2(d + X_COL, pack2(r0.y, r1.y), pack2(r2.y, r3.y));
      sts_2x2(d + 2 * X_COL, pack2(r0.z, r1.z), pack2(r2.z, r3.z));
      sts_2x2(d + 3 * X_COL, pack2(r0.w, r1.w), pack2(r2.w, r3.w));
    };
    if (have_cache && nsl >= nst) {
      // every stream of the tile has its own landing slot: wait for all of them (they were requested a block ago), move
      // everything in ONE flat loop, signal the group, and only then recycle the slots -- one latency chain per block
      // instead of one per stream (the per-stream version kept the group waiting on halo_bar 10-17 % of the time)
      for (int m = 0; m < nst; ++m) {
        const uint32_t use = (uint32_t)(k + m);
        mbar_wait(&B.stg_bar[slot0 + use % nsl], (use / nsl) & 1);
      }
      TPH(t_stg)
      const int per = 16 << lgg;
#pragma unroll 1
      for (int it = lane; it < nst * per; it += 32) {
        const int m = it >> (4 + lgg);
        move_item(STG + (slot0 + (uint32_t)(k + m) % nsl) * STG_FLOATS, (sg0 + m) * Lw + PADR - pad, it & (per - 1));
      }
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&B.halo_bar[i]);               // the tile's slices of this block are in place
        fence_proxy_async();                       // the slots were read through the generic proxy; TMA rewrites them
        for (int m = 0; m < nst; ++m)
          if (k + m + nsl < njobs) issue_tma(k + m + nsl);
      }
      k += nst;
      TPH(t_tr)
      continue;
    }
    for (int sg = sg0; sg < sg0 + nst; ++sg, ++k) {
      const int colb = sg * Lw + PADR - pad;       // first cache column of this stream for this block
      if (have_cache) {
        const uint32_t use = (uint32_t)k, slot = slot0 + use % nsl;
        if (lane == 0) mbar_wait_backoff(&B.stg_bar[slot], (use / nsl) & 1);
        __syncwarp();
        const float* slotp = STG + slot * STG_FLOATS;
#pragma unroll 1
        for (int it = lane; it < (16 << lgg); it += 32) move_item(slotp, colb, it);
        __syncwarp();                              // every lane has read the slot
        if (lane == 0 && k + nsl < njobs) {        // refill it: the same ring position, nsl jobs ahead
          fence_proxy_async();                     // the slot was read through the generic proxy; TMA rewrites it
          issue_tma(k + nsl);
        }
      } else {
        const f32x2 z = 0ull;
#pragma unroll 1
        for (int e = lane; e < pad * 16; e += 32) sts_2x2(x_addr(xs, colb + (e >> 4), 4 * (e & 15)), z, z);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&B.halo_bar[i]);    // the tile's slices of this block are in place
    TPH(t_tr)
  }
#if MDTC_TIMING
  if (blockIdx.x == 0 && lane == 0) printf("loader %d: wait h_free %lld, wait landing %lld, transposes %lld (nsl %d)\n", i, t_hf, t_stg, t_tr, nsl);
#endif
  // DW of the last block still signals h_free: consume it so the parity stays in step
  if (lane == 0) mbar_wait_backoff(&B.h_free[i], hf_par & 1);
  hf_par ^= 1u;
}

// KT: compile-time tap count (5 = every shipped mdtc config; 0 = read a.ktaps, taps guarded one by one)
// HEAD: utterance-level head variant: instead of the per-frame classifier, every stream's stack-output sum is summed over
// frames [a.pool_t0, a.pool_t1) into a.pool (B, 64); cls_head.cu applies the MLP
template <int KT, bool HEAD>
__global__ void __launch_bounds__(NT_TC, 1) mdtc_tc_kernel(const __grid_constant__ TcArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
  __shared__ uint64_t halo_bar[NG], h_free[NG];
  __shared__ uint64_t w_bar[2], w_free[2], stg_bar[NSLOT];
  constexpr int nslot = HEAD ? NSLOT_HEAD : NSLOT;

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // warp-uniform for the compiler too (no divergence regions around the roles)
  const int T = a.T, K = KT ? KT : a.ktaps;
  const float* vec = a.vec;

  uint32_t sbase;                                  // shared-window address of `base`, pinned in a register
  asm volatile("mov.u32 %0, %1;" : "=r"(sbase) : "r"(smem_u32(base)));
  const uint32_t xs = sbase + OFF_X;

  if (tid == 0) {
    for (int i = 0; i < NG; ++i) { mbar_init(&halo_bar[i], 1); mbar_init(&h_free[i], WPG); }
    for (int i = 0; i < 2; ++i) { mbar_init(&w_bar[i], 1); mbar_init(&w_free[i], NCW); }
    mbar_fence_init();
  }
  if constexpr (!HEAD) {
    // the classifier weights in shared memory: the stack-end partial sums read them right after each residual store,
    // where a global load's latency is exposed once per fragment column (measured: 15 % of the flagship step)
    float* wcs = reinterpret_cast<float*>(base + OFF_WC);
    for (int i = tid; i < C * a.odim; i += NT_TC) wcs[i] = __ldg(vec + a.v_wc + i);
  }
  __syncthreads();
  const Bars bars{halo_bar, h_free, w_bar, w_free, stg_bar};
  // phase parities: every waiter keeps its own copy; all copies of a barrier advance in lock step
  uint32_t halo_par = 0;                                             // compute groups
  uint32_t hf_par = 0;                                               // loaders: bit i = tile i
  uint32_t w_par = 0, wf_par = 0;                                    // bit s = slot s
  const int natoms = (a.idim + 63) / 64;
  const int PADR = a.padr, Lw = a.padr + T;
  const int spt = a.spt;                                             // streams per tile

  // balanced contiguous partition of the streams over the grid
  const int sb = (int)(((long long)a.B * blockIdx.x) / gridDim.x);
  const int se = (int)(((long long)a.B * (blockIdx.x + 1)) / gridDim.x);
  int done = sb, b0 = 0, ns = 0, ntile = 0;
  // opens the next pass: every thread of the CTA calls it once per pass, so the __syncthreads stay in step
  auto begin_pass = [&]() {
    const int remaining = se - done;
    const int passes_left = (remaining + a.smax - 1) / a.smax;
    ns = (remaining + passes_left - 1) / passes_left;                 // streams of this pass (resident in X)
    b0 = done;
    done += ns;
    ntile = (ns + spt - 1) / spt;
    // the landing slots are dealt out per pass (by stream count): their barriers start every pass from phase 0
    if (tid == 0) {
      for (int i = 0; i < nslot; ++i) mbar_init(&stg_bar[i], 1);
      mbar_fence_init();
    }
    __syncthreads();
  };
  auto tile_streams = [&](int i) { return min(spt, ns - i * spt); };  // streams of tile i (sequential fill)

  // The register handoff is warpgroup-collective: every warp of a warpgroup executes it once, before its pass loop.
  // ptxas honours the new limits only in code that the other side never runs, so each side has its own pass loop.
  if (warp < NCW) {
    setmaxnreg_inc<REG_COMPUTE>();
    while (done < se) {
      begin_pass();
      // ================================================================== COMPUTE GROUPS (WPG warps per tile)
      // warp = grp * WPG + 4 wg + w: warpgroup wg of the tile owns rows [64 wg, 64 wg + 64) and runs their GEMMs; a thread
      // holds the wgmma fragment of rows r0 and r0 + 8 (r0 = 64 wg + 16 w + lane / 4), channel pairs 8 m + 2 (lane % 4)
      const int grp = warp / WPG, wq = warp % WPG;
      // live warps of the group: a tile of <= 64 rows leaves warpgroup 1 without a row (the flagship 1024 x 40 shape
      // runs its 8-stream CTAs as two passes of 3 + 1 streams, so every pass has one), and that warpgroup skips the
      // depthwise conv, the GEMMs and the epilogues.  The head variant keeps all eight: its pooling splits the
      // channels over the group's warps.
      const int nlw = (grp < ntile && !HEAD && tile_streams(grp) * T <= 64) ? WPG / 2 : WPG;
      if (grp < ntile && wq < nlw) {
        const int nst = tile_streams(grp), rows = nst * T;
        const int q4 = lane & 3, r0 = 64 * (wq >> 2) + 16 * (wq & 3) + (lane >> 2);
        bool live[2];
        int col[2], sgr[2], ttr[2];
        uint32_t t_own[2];                                 // X address of the row's channel pair 2 q4 (chunk 0)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r0 + 8 * h;
          live[h] = row < rows;
          const int s = live[h] ? row / T : 0;
          ttr[h] = live[h] ? row - s * T : 0;
          sgr[h] = grp * spt + s;                          // stream index inside the pass
          col[h] = sgr[h] * Lw + PADR + ttr[h];            // this row's frame column (dead rows alias a valid one)
          t_own[h] = x_addr(xs, col[h], 2 * q4);
        }
        const float* cwf = reinterpret_cast<const float*>(&a.cw[0][0]);
        constexpr int CWS = 7 * 64;                        // floats per block in cw
        float part[2][8];                                  // classifier partial sums of the two rows
        if constexpr (!HEAD) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int j = 0; j < 8; ++j) part[h][j] = 0.f;
        }
        float acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        uint32_t ahi[4][4], alo[4][4];                     // A fragments of the 4 K steps of a 64-wide GEMM

        uint64_t dW_hi[2], dW_lo[2];
#pragma unroll
        for (int sl = 0; sl < 2; ++sl) {
          dW_hi[sl] = make_sdesc_sw128(sbase + OFF_W + sl * W_SLOT);
          dW_lo[sl] = make_sdesc_sw128(sbase + OFF_W + sl * W_SLOT + 8192);
        }
        // waits for this warpgroup's MMAs and releases their weight slot
        auto gemm_finish = [&](int slot) {
          wgmma_wait<0>();
          wgmma_reg_fence(acc);
          __syncwarp();
          if (lane == 0) mbar_arrive(&w_free[slot]);
        };
        // 3-pass bf16x3 GEMM acc (+)= A * W^T over weight slot `slot` (waited for here); with finish == false the MMAs
        // are left in flight, and the caller runs gemm_finish once its own work under them is done
        auto gemm = [&](int slot, int ksteps, bool fresh, bool finish = true) {
          mbar_wait(&w_bar[slot], (w_par >> slot) & 1);
          w_par ^= 1u << slot;
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_rs(acc, ahi[k][0], ahi[k][1], ahi[k][2], ahi[k][3], dW_hi[slot] + 2 * k, (fresh && k == 0) ? 0u : 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_rs(acc, alo[k][0], alo[k][1], alo[k][2], alo[k][3], dW_hi[slot] + 2 * k, 1u);
#pragma unroll
          for (int k = 0; k < 4; ++k)
            if (k < ksteps) wgmma_m64n64k16_rs(acc, ahi[k][0], ahi[k][1], ahi[k][2], ahi[k][3], dW_lo[slot] + 2 * k, 1u);
          wgmma_commit();
          if (finish) gemm_finish(slot);
        };

        // ---- features (+CMVN) -> bf16x3 A fragments, first Linear over slot 0 (K 0..63) and slot 1 (K 64..)
        for (int at = 0; at < natoms; ++at) {
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
              split_pair_rn(pack2(v0, v1), ahi[k][p], alo[k][p]);
            }
          const int rem = a.idim - 64 * at;
          gemm(at, rem >= 64 ? 4 : (rem + 15) >> 4, at == 0);
        }
        // ---- x = relu(D + bp) -> X                                            (subsampling.py:53-57)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(vec + a.v_bp + 8 * j + 2 * q4));
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (live[h])
              sts_f2(t_own[h] + 16u * j, fmaxf(acc[4 * j + 2 * h] + b.x, 0.f), fmaxf(acc[4 * j + 2 * h + 1] + b.y, 0.f));
        }
        group_barrier(grp, nlw);                // X of the tile complete before the first depthwise conv reads across rows

#if MDTC_TIMING
        // halo wait, depthwise conv, cache stores, GEMM1 (incl. weight wait), epilogue 1, GEMM2, first barrier,
        // epilogue 2, second barrier
        long long t_halo = 0, t_dw = 0, t_cache = 0, t_g1 = 0, t_e1 = 0, t_g2 = 0, t_bar1 = 0, t_e2 = 0, t_bar2 = 0;
        long long t_last_ = clock64();
#endif
        // ---- blocks
        for (int blk = 0; blk < a.nblocks; ++blk) {
          const int d = a.dil[blk], pad = d * (K - 1);
          const bool stack_end = (blk > 0) && (blk % a.stack_size == 0);
          const float* cwb = cwf + blk * CWS;
          // ---------------- depthwise dilated conv (+folded BN) -> A fragments                 (mdtc.py:56-57)
          mbar_wait(&halo_bar[grp], halo_par);
          halo_par ^= 1;
          TPH(t_halo)
          {
            uint32_t tj[2][5];
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int j = 0; j < 5; ++j) {
                tj[h][j] = x_addr(xs, col[h] - pad + j * d, 2 * q4);
              }
#pragma unroll
            for (int k = 0; k < 4; ++k)
#pragma unroll
              for (int p = 0; p < 4; ++p) {
                const int h = p & 1, m = 2 * k + (p >> 1), ch = 8 * m + 2 * q4;
                // (the folded depthwise bias is not added here: the host folds it through the pointwise-1 matrix into
                // b1, model_host.cu pack_tc)
                float s0 = 0.f, s1 = 0.f;
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                  if (KT ? j < KT : j < K) {
                    const float2 x = lds_f2(tj[h][j] + 16u * m);
                    s0 = fmaf(x.x, cwb[64 * j + ch], s0);
                    s1 = fmaf(x.y, cwb[64 * j + ch + 1], s1);
                  }
                }
                split_pair_rn(pack2(s0, s1), ahi[k][p], alo[k][p]);
              }
          }
          // this warp is done with the block's cache columns in front of the frames: when the new cache slice is made of
          // frame columns only (T >= pad) the loader may start transposing the next block's slices now, not after the
          // stores below (which read those columns when T < pad)
          TPH(t_dw)
          const bool early_free = T >= pad;
          __syncwarp();
          if (early_free && lane == 0) mbar_arrive(&h_free[grp]);
          // ---------------- new cache slices of this tile: out_cache[b][c][off + j] = cat[c][T + j] (mdtc.py:113).
          // A warp reads jpl columns x 32 / jpl channel quads per request; 8 lanes write 32 contiguous bytes of one
          // cache row.  Quad cq = 2 m + h takes the chunk index m = q >> 1 rotated left by one bit, so the chunks of one
          // request spread over the bank groups (col + m) mod 8: conflict-free for 4- and 8-column slices too.
          {
            const int off = a.coff[blk];
            const int jpl = pad < 32 ? pad : 32, lgj = 31 - __clz(jpl), qstep = 32 >> lgj;
            const int j = lane & (jpl - 1), qs = lane >> lgj, per = 16 >> (5 - lgj);      // quads passes per stream
            const int nitem = nst * per;
            for (int it = wq; it < nitem; it += nlw) {
              const int s2 = it / per, q = (it - s2 * per) * qstep + qs, mq = q >> 1;
              const int cq = 2 * (((mq << 1) | (mq >> 2)) & 7) + (q & 1);
              const int sg2 = grp * spt + s2;
              const uint32_t src = x_addr(xs, sg2 * Lw + PADR + T - pad + j, 4 * cq);
              f32x2 v01, v23;
              lds_2x2(src, v01, v23);
              float v0, v1, v2, v3;
              unpack2(v01, v0, v1);
              unpack2(v23, v2, v3);
              float* g = a.out_cache + ((size_t)(b0 + sg2) * C + 4 * cq) * a.P + off + j;
              g[0] = v0; g[a.P] = v1; g[2 * a.P] = v2; g[3 * a.P] = v3;
            }
            if (!early_free) {
              __syncwarp();
              if (lane == 0) mbar_arrive(&h_free[grp]);    // the tile's cache columns may be overwritten
            }
          }
          TPH(t_cache)
          // ---------------- pointwise-1 GEMM, h = relu(D + b1) -> A fragments                 (mdtc.py:115)
          // The per-block biases are lane-indexed reads of the parameter bank (four addresses per warp).  Each wait in
          // gemm clobbers memory, so a read written after it cannot move above it and its latency is exposed; read
          // before the GEMM, it completes under the MMAs (measured: 2.6 % of the flagship step).
          float2 b1[8];                         // pointwise-1 bias of channels 8 j + 2 q4, + 1
#pragma unroll
          for (int j = 0; j < 8; ++j) b1[j] = make_float2(cwb[5 * 64 + 8 * j + 2 * q4], cwb[5 * 64 + 8 * j + 2 * q4 + 1]);
          gemm(0, 4, true);
          TPH(t_g1)
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              const int i = 8 * k + 2 * p;
              const float2 b = b1[2 * k + (p >> 1)];      // channels 16 k + 8 (p >> 1) + 2 q4, + 1
              split_pair_rz_relu(pack2(acc[i] + b.x, acc[i + 1] + b.y), ahi[k][p], alo[k][p]);
            }
          // ---------------- pointwise-2 GEMM; x' = relu(D + b2 + x) -> X; classifier partial sums at the end of a stack
          TPH(t_e1)
          float2 b2[8];                         // pointwise-2 bias of channels 8 j + 2 q4, + 1
#pragma unroll
          for (int j = 0; j < 8; ++j) b2[j] = make_float2(cwb[6 * 64 + 8 * j + 2 * q4], cwb[6 * 64 + 8 * j + 2 * q4 + 1]);
          gemm(1, 4, true, false);                                             // (mdtc.py:116-118, 266-273)
          TPH(t_g2)
          group_barrier(grp, nlw);              // every row's depthwise taps and cache stores have read x (under the MMAs)
          TPH(t_bar1)
          gemm_finish(1);
          // the rows' residual x, read before the first x' store: the loads are volatile asm like the stores, so read
          // column by column each load would wait for the previous column's store and every column would pay a full
          // shared-memory round trip.  Each address is the thread's own, so the order changes no value.
          float2 res[8][2];
#pragma unroll
          for (int j = 0; j < 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) res[j][h] = lds_f2(t_own[h] + 16u * j);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int ch = 8 * j + 2 * q4;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const uint32_t ax = t_own[h] + 16u * j;
              const float2 r = res[j][h];
              const float o0 = fmaxf(acc[4 * j + 2 * h] + b2[j].x + r.x, 0.f);
              const float o1 = fmaxf(acc[4 * j + 2 * h + 1] + b2[j].y + r.y, 0.f);
              if (live[h]) sts_f2(ax, o0, o1);
              if (!HEAD && stack_end) {
                // the classifier is linear: W_c (sum of stack outputs) = sum of W_c (stack output)
                const float* wc = reinterpret_cast<const float*>(base + OFF_WC) + ch * a.odim;
#pragma unroll
                for (int jo = 0; jo < 8; ++jo)
                  if (jo < a.odim) part[h][jo] = fmaf(wc[a.odim + jo], o1, fmaf(wc[jo], o0, part[h][jo]));
              }
            }
          }
          TPH(t_e2)
          group_barrier(grp, nlw);              // x' of every row of the tile complete before the next block's conv
          TPH(t_bar2)
          if constexpr (HEAD) {
            // X now holds the stack output of every frame of the tile, and stays so until the next block's second
            // group barrier.  Warp wq sums channels 8 wq .. 8 wq + 7; lane = 8 q + channel, q = frame phase mod 4:
            // strided frame sums, two shuffles in a fixed order, then the q = 0 lane keeps the stream's running sum
            // over the stacks in the shared pool buffer (always the same thread: no barrier, no atomics)
            if (stack_end && a.pool_t1 > a.pool_t0) {
              const int c = 8 * wq + (lane & 7), q = lane >> 3;
              float* pl = reinterpret_cast<float*>(base + OFF_POOL) + grp * POOL_SPT * C;
              for (int s2 = 0; s2 < nst; ++s2) {
                const int colb = (grp * spt + s2) * Lw + PADR;
                float v = 0.f;
                for (int t = a.pool_t0 + q; t < a.pool_t1; t += 4) {
                  float x;
                  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(x_addr(xs, colb + t, c)));
                  v += x;
                }
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (q == 0) pl[s2 * C + c] = (blk == a.stack_size) ? v : pl[s2 * C + c] + v;
              }
            }
          }
        }
#if MDTC_TIMING
        if (blockIdx.x == 0 && wq == 0 && lane == 0)
          printf("group %d (%d rows, pass at stream %d): halo %lld dw %lld cache %lld gemm1 %lld epi1 %lld gemm2 %lld "
                 "bar1 %lld epi2 %lld bar2 %lld\n", grp, rows, b0, t_halo, t_dw, t_cache, t_g1, t_e1, t_g2, t_bar1, t_e2,
                 t_bar2);
#endif
        if constexpr (HEAD) {
          // the stream's pooled vector: the first time-chunk of the call stores, later ones add (stream-ordered launches)
          if (a.pool_t1 > a.pool_t0 && lane < 8) {
            const int c = 8 * wq + lane;
            const float* pl = reinterpret_cast<const float*>(base + OFF_POOL) + grp * POOL_SPT * C;
            for (int s2 = 0; s2 < nst; ++s2) {
              float* g = a.pool + (size_t)(b0 + grp * spt + s2) * C + c;
              *g = a.pool_add ? *g + pl[s2 * C + c] : pl[s2 * C + c];
            }
          }
        } else {
        // ---- classifier bias + activation: the four lanes of a row hold disjoint channel pairs
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int jo = 0; jo < 8; ++jo) {
            part[h][jo] += __shfl_xor_sync(0xffffffffu, part[h][jo], 1);
            part[h][jo] += __shfl_xor_sync(0xffffffffu, part[h][jo], 2);
          }
          if (live[h] && q4 == 0) {
            float* o = a.out + (size_t)(b0 + sgr[h]) * a.out_bstride + (size_t)ttr[h] * a.odim;
#pragma unroll
            for (int jo = 0; jo < 8; ++jo) {
              if (jo < a.odim) {
                float y = part[h][jo] + __ldg(vec + a.v_bc + jo);
                if (a.act == WEKWS_ACT_SIGMOID) y = sigmoidf_acc(y);
                o[jo] = y;
              }
            }
          }
        }
        }  // !HEAD
      } else {
        // a group without streams in this pass, or a warpgroup without rows in a live tile, still releases every
        // weight slot use (w_free counts every compute warp's arrival); all lanes keep the same phase bookkeeping
        const bool in_tile = grp < ntile;
        mbar_wait(&w_bar[0], w_par & 1);
        if (lane == 0) mbar_arrive(&w_free[0]);
        if (natoms > 1) {
          mbar_wait(&w_bar[1], (w_par >> 1) & 1);
          if (lane == 0) mbar_arrive(&w_free[1]);
        }
        w_par ^= natoms > 1 ? 3u : 1u;
        for (int blk = 0; blk < a.nblocks; ++blk)
          for (int job = 0; job < 2; ++job) {
            mbar_wait(&w_bar[job], (w_par >> job) & 1);
            w_par ^= 1u << job;
            if (lane == 0) mbar_arrive(&w_free[job]);
            // in a live tile it also stands in for its share of h_free (WPG arrivals per block).  Arriving only once
            // W1 of the block has landed keeps it in step: W1(blk + 1) is loaded only after every live warp's
            // pointwise-1 GEMM of blk, and each live warp arrives on h_free(blk) before that GEMM.
            if (job == 0 && in_tile && lane == 0) mbar_arrive(&h_free[grp]);
          }
        if (in_tile) halo_par ^= (uint32_t)a.nblocks & 1u;   // the tile's halo_bar went through nblocks phases
      }
      __syncthreads();     // pass boundary: X, the landing slots and the rings are reused
    }
  } else {
    setmaxnreg_dec<REG_SERVICE>();
    while (done < se) {
      begin_pass();
      if (warp == W_WGT) {
        if (lane == 0) weights_role(a, base, bars, K, natoms, wf_par, b0 == sb);
      } else if (warp < W_LD + NG) {
        loader_role(a, base, bars, warp - W_LD, lane, K, ns, b0, ntile, nslot, hf_par);
      }
      __syncthreads();     // pass boundary
    }
  }
}

}  // namespace

bool tc_eligible(const TcArgs& a, int padmax, bool head) {
  // first Linear: at most two A atoms, K <= 96; the per-frame classifier keeps odim <= 8 partial sums per row
  if (a.idim % 8 != 0 || a.idim > 96 || (!head && a.odim > 8) || a.ktaps > 5) return false;
  if (a.nblocks > kTcMaxBlocks) return false;                                        // taps / biases travel in the parameter block
  if (padmax > 32 || a.P % 4 != 0) return false;
  for (int b = 0; b < a.nblocks; ++b)
  {
    const int pad = a.dil[b] * (a.ktaps - 1);
    if (pad < 4 || (pad & (pad - 1)) != 0 || a.coff[b] % 4 != 0) return false;   // power-of-two slices, 16-byte aligned
  }
  return true;
}

int tc_max_T() { return 128; }

namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}
}  // namespace

int mdtc_tc_launch(TcArgs a, int padmax, cudaStream_t st, bool head) {
  WEKWS_REQUIRE(a.T >= 1 && a.T <= 128 && a.B >= 1, "mdtc_tc_launch: bad shape");
  a.padr = (padmax + 3) & ~3;
  const int Lw = a.padr + a.T;
  a.spt = 128 / a.T;                                   // streams per 128-row tile
  WEKWS_REQUIRE(a.spt >= 1 && Lw <= XCOLS, "mdtc_tc_launch: tile does not fit");
  WEKWS_REQUIRE(!head || (a.pool != nullptr && a.spt <= POOL_SPT), "mdtc_tc_launch: bad head call");
  int smax = NG * a.spt;                               // streams resident per pass
  if (smax > XCOLS / Lw) smax = XCOLS / Lw;
  a.smax = smax;
  // tensor maps over the incoming cache (B*64 rows of P floats): one per distinct slice width
  if (a.in_cache != nullptr) {
    EncodeTiledFn enc = encode_tiled_fn();
    WEKWS_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled is not available from this driver");
    int pads[4], npads = 0;
    for (int b = 0; b < a.nblocks; ++b) {
      const int pad = a.dil[b] * (a.ktaps - 1);
      int i = 0;
      while (i < npads && pads[i] != pad) ++i;
      if (i == npads) {
        WEKWS_REQUIRE(npads < 4, "more than 4 distinct cache slice widths");
        pads[npads++] = pad;
        const cuuint64_t gdim[2] = {(cuuint64_t)a.P, (cuuint64_t)a.B * C};
        const cuuint64_t gstr[1] = {(cuuint64_t)a.P * sizeof(float)};
        const cuuint32_t box[2] = {(cuuint32_t)pad, (cuuint32_t)C};
        const cuuint32_t estr[2] = {1, 1};
        const CUresult rc = enc(&a.tmap[i], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(a.in_cache), gdim,
                                gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        WEKWS_REQUIRE(rc == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)rc);
      }
      a.tmap_idx[b] = i;
    }
  }
  const int sms = device_sm_count();
  const int grid = a.B < sms ? a.B : sms;
  auto* kernel = head ? (a.ktaps == 5 ? mdtc_tc_kernel<5, true> : mdtc_tc_kernel<0, true>)
                      : (a.ktaps == 5 ? mdtc_tc_kernel<5, false> : mdtc_tc_kernel<0, false>);
  const int smem = head ? SMEM_TOTAL_HEAD : SMEM_TOTAL;
  if (const int rc = opt_in_smem((const void*)kernel, smem)) return rc;
  kernel<<<grid, NT_TC, smem, st>>>(a);
  return check_launch("mdtc_tc_kernel");
}

}  // namespace wekws
