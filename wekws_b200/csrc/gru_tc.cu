// Tensor-core GRU forward with weight streaming (KWSModel.forward with the GRU backbone, kws_model.py:128-133; PyTorch
// gate order r, z, n -- see gru.cu for the FP32 kernel of the same math).
//
// Shape of the problem at the streaming operating point (B = 512 streams, one frame per call): 0.2 GFLOP against 786 KB
// of weights.  Here a CTA owns a tile of up to 64 streams and the GEMMs are TRANSPOSED: D^T[gate row][stream] =
// W[gate row][k] * X^T[k][stream], i.e. the weights are the M operand (one gate of all 128 hidden units, streamed from
// L2 through a ring of 16 KB pre-swizzled bf16 hi|lo chunks by bulk async copies), the activations are the N = 64
// operand (K-major SWIZZLE_128B images in shared memory: features, x0, h of each layer, each split into bf16 hi + lo
// once by its producer).  Two warpgroups own 64 hidden units each; a gate's accumulator (64 units x 64 streams fp32)
// lives in the registers of its warpgroup, so the gate math runs where the accumulator is and the old h stays in fp32
// registers for the whole call.  fp32 parity through the bf16 x3 split (W_hi X_hi + W_hi X_lo + W_lo X_hi, fp32
// accumulate).  Gates are computed one after the other (r, n_h, n_x, z: two accumulators live at a time), in the order
// the host packs the weight stream.
//
// Per step and CTA: (2 ceil(idim/64) + 24 L) weight chunks = 786 KB for the shipped model.
//
// Warps (352 threads): 0-7 unit owners (warpgroup = 64 hidden units): GEMMs, epilogues, gate math, classifier, cache
// I/O; 8 weight ring (one lane); 9-10 feature rows -> operand image for the next step.
#include "common.cuh"
#include "gru_tc.h"
#include "tc_common.cuh"

namespace wekws {
namespace {

using namespace tc;

constexpr int M = 64;                   // streams per CTA tile (the MMA N)
constexpr int H = 128;                  // hidden units (the MMA M of the two warpgroups)
constexpr int NOW = 8;                  // unit-owner warps
constexpr int NT = (NOW + 3) * 32;
constexpr int SLAB = M * 128;           // one activation K-slab image (64 rows x 128 B), 8 KB
constexpr int IMG = 4 * SLAB;           // activation image: [slab 0 hi][slab 0 lo][slab 1 hi][slab 1 lo]
constexpr int CHUNK = H * 128;          // one weight chunk: 128 gate rows x 64 K, bf16, 16 KB
constexpr int NSLOT = 5;
// shared memory map (bytes, 1024-aligned)
constexpr int OFF_F = 0;                // feature image (K = idim <= 128)
constexpr int OFF_X0 = OFF_F + IMG;     // x0 = relu(Linear)
constexpr int OFF_H = OFF_X0 + IMG;     // h of layer l at OFF_H + l * IMG
constexpr int OFF_RING = OFF_H + 2 * IMG;
constexpr int OFF_END = OFF_RING + NSLOT * CHUNK;
constexpr int SMEM_BYTES = OFF_END + 1024;
static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a CTA may use");

// byte offset of K element k (0..127) of stream row m inside an activation image (hi; lo at + SLAB)
__device__ __forceinline__ uint32_t a_off(int m, int k) {
  return (uint32_t)((k >> 6) * 2 * SLAB + m * 128 + ((((k & 63) >> 3) ^ (m & 7)) << 4) + (k & 7) * 2);
}
__device__ __forceinline__ void split1(float x, uint16_t& hi, uint16_t& lo) {
  const __nv_bfloat16 h = __float2bfloat16_rn(x);
  const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
  hi = *reinterpret_cast<const uint16_t*>(&h);
  lo = *reinterpret_cast<const uint16_t*>(&l);
}
// Gates on the SFU approximations (ex2.approx, rcp.approx: ~1 ulp each): absolute error ~1e-7, far inside the
// fp32-parity budget (posterior 1e-4), and ~25 instructions per (unit, stream) instead of ~80 with expf / tanhf / IEEE
// division -- the gate math is on the critical path of every step.
__device__ __forceinline__ float ex2_fast(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_fast(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
constexpr float LOG2E = 1.4426950408889634f;
// sigmoid(g + b) with nb = -b * log2(e) folded by the caller: 1 / (1 + 2^(-(g + b) log2 e))
__device__ __forceinline__ float sigmoid_fast(float g, float nb) { return rcp_fast(1.f + ex2_fast(fmaf(g, -LOG2E, nb))); }
// tanh(t) = 1 - 2 / (1 + 2^(2 t log2 e)); the exponent is clamped so that 2^x stays finite (tanh is 1 there anyway)
__device__ __forceinline__ float tanh_fast(float t) {
  return fmaf(-2.f, rcp_fast(1.f + ex2_fast(fminf(t * (2.f * LOG2E), 126.f))), 1.f);
}
__device__ __forceinline__ void owner_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(NOW * 32) : "memory"); }

struct Bars {
  uint64_t w_full[NSLOT], w_free[NSLOT];
  uint64_t f_rdy, lin_bar;
};

__device__ __forceinline__ void wait_flip(uint64_t* bar, uint32_t& par) {
  mbar_wait(bar, par);
  par ^= 1;
}

// ---------------------------------------------------------------------------------------------- weight ring (one lane)
__device__ __noinline__ void weights_role(const GruTcArgs& a, Bars* b, uint8_t* base, int my_tiles) {
  const int per_step = 2 * ((a.idim + 63) >> 6) + 24 * a.L;
  const long long total = (long long)my_tiles * a.T * per_step;
  int ci = 0;
  uint32_t slot = 0, free_par = 0;
  for (long long c = 0; c < total; ++c) {
    if (c >= NSLOT) {
      mbar_wait(&b->w_free[slot], (free_par >> slot) & 1u);
      free_par ^= 1u << slot;
    }
    mbar_arrive_expect_tx(&b->w_full[slot], CHUNK);
    bulk_g2s(base + OFF_RING + slot * CHUNK, a.wimg + (size_t)ci * CHUNK, CHUNK, &b->w_full[slot]);
    slot = slot + 1 == NSLOT ? 0 : slot + 1;
    ci = ci + 1 == per_step ? 0 : ci + 1;
  }
}

// Consumer side of the weight ring, run by every unit-owner warp (each warpgroup reads its 64 rows of every chunk)
struct Ring {
  Bars* b;
  uint32_t ring0;                          // shared address of slot 0 + this warpgroup's row offset
  uint32_t slot, full_par, held[4], nheld;
  __device__ __forceinline__ uint64_t take() {             // wait for the next chunk, return its descriptor
    mbar_wait(&b->w_full[slot], (full_par >> slot) & 1u);
    full_par ^= 1u << slot;
    held[nheld++] = slot;
    const uint64_t d = make_sdesc_sw128(ring0 + slot * CHUNK);
    slot = slot + 1 == NSLOT ? 0 : slot + 1;
    return d;
  }
  // wait for the issued MMAs, then free the chunks they read
  __device__ __forceinline__ void finish(float (&acc)[32]) {
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(acc);
    __syncwarp();
    if ((threadIdx.x & 31) == 0)
      for (uint32_t i = 0; i < nheld; ++i) mbar_arrive(&b->w_free[held[i]]);
    nheld = 0;
  }
  // one K slab with `ksteps` K steps: acc (+)= W[:, slab] X[:, slab]^T with the x3 split (hi chunk, then lo chunk)
  __device__ __forceinline__ void slab(float (&acc)[32], uint64_t xhi, int ksteps, bool fresh) {
    const uint64_t xlo = xhi + (SLAB >> 4);
    const uint64_t whi = take();
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < ksteps) wgmma_m64n64k16_ss(acc, whi + 2 * k, xhi + 2 * k, (fresh && k == 0) ? 0u : 1u);
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < ksteps) wgmma_m64n64k16_ss(acc, whi + 2 * k, xlo + 2 * k, 1u);
    const uint64_t wlo = take();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < ksteps) wgmma_m64n64k16_ss(acc, wlo + 2 * k, xhi + 2 * k, 1u);
  }
  // one gate block over K = 128 (two slabs), waited for; FRESH: the first MMA overwrites acc
  __device__ __forceinline__ void gate(float (&acc)[32], uint64_t ximg, bool fresh) {
    slab(acc, ximg, 4, fresh);
    slab(acc, ximg + (uint64_t)(2 * SLAB >> 4), 4, false);
    finish(acc);
  }
};

// ------------------------------------------------------------------------------------------------------------- kernel
__global__ void __launch_bounds__(NT, 1) gru_tc_kernel(const __grid_constant__ GruTcArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = smem_raw + ((1024 - (smem_u32(smem_raw) & 1023)) & 1023);
  __shared__ Bars bars;
  const uint32_t sbase = smem_u32(base);
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const float* vec = a.vec;
  const int L = a.L, T = a.T;

  if (tid == 0) {
    for (int i = 0; i < NSLOT; ++i) { mbar_init(&bars.w_full[i], 1); mbar_init(&bars.w_free[i], NOW); }
    mbar_init(&bars.f_rdy, 2);
    mbar_init(&bars.lin_bar, NOW);
    mbar_fence_init();
  }
  // the feature image's K padding must be finite (it meets zero weights): clear it once
  for (int i = tid; i < IMG / 16; i += NT) reinterpret_cast<uint4*>(base + OFF_F)[i] = make_uint4(0, 0, 0, 0);
  fence_proxy_async();
  __syncthreads();

  const int my_tiles = a.n_tiles > (int)blockIdx.x ? (a.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;

  if (warp == NOW) {
    if (lane == 0) weights_role(a, &bars, base, my_tiles);
  } else if (warp > NOW) {
    // ---- feature rows: thread = stream row; CMVN (cmvn.py:45-47), bf16 hi|lo split, 16-byte chunks into the image
    const int m = tid - (NOW + 1) * 32;
    uint32_t p_lin = 0;
    long long step = 0;
    for (int it = 0; it < my_tiles; ++it) {
      const int b0 = (blockIdx.x + it * gridDim.x) * a.ms;
      const bool live = m < a.ms && b0 + m < a.B;
      for (int t = 0; t < T; ++t, ++step) {
        float4 f4[24];
        const float* src0 = a.feats + ((size_t)(b0 + m) * T + t) * a.idim;
        const bool vec4 = (a.idim & 3) == 0 && (reinterpret_cast<uintptr_t>(a.feats) & 15) == 0;
#pragma unroll
        for (int i = 0; i < 24; ++i) {
          f4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (live && 4 * i < a.idim) {
            if (vec4) f4[i] = __ldg(reinterpret_cast<const float4*>(src0) + i);
            else {
              f4[i].x = __ldg(src0 + 4 * i);
              if (4 * i + 1 < a.idim) f4[i].y = __ldg(src0 + 4 * i + 1);
              if (4 * i + 2 < a.idim) f4[i].z = __ldg(src0 + 4 * i + 2);
              if (4 * i + 3 < a.idim) f4[i].w = __ldg(src0 + 4 * i + 3);
            }
          }
        }
        if (step > 0) wait_flip(&bars.lin_bar, p_lin);     // the previous step's Linear has read the image
#pragma unroll
        for (int ch = 0; ch < 12; ++ch) {
          if (8 * ch < a.idim) {
            float v[8] = {f4[2 * ch].x, f4[2 * ch].y, f4[2 * ch].z, f4[2 * ch].w,
                          f4[2 * ch + 1].x, f4[2 * ch + 1].y, f4[2 * ch + 1].z, f4[2 * ch + 1].w};
            const int k0 = 8 * ch;
            if (a.has_cmvn && live) {
#pragma unroll
              for (int u = 0; u < 8; ++u)
                if (k0 + u < a.idim) v[u] = (v[u] - __ldg(vec + a.v_mean + k0 + u)) * __ldg(vec + a.v_istd + k0 + u);
            }
            const uint32_t off = a_off(m, k0);
            split_store8(v, base + OFF_F, base + OFF_F + SLAB, off);
          }
        }
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars.f_rdy);
      }
    }
  } else {
    // ---- unit owners: warpgroup wg = hidden units [64 wg, 64 wg + 64); a thread holds the wgmma fragment of units
    // u0 and u0 + 8 (u0 = 64 wg + 16 (warp % 4) + lane / 4) x streams 8 jj + 2 (lane % 4) + e
    const int wg = warp >> 2, q4 = lane & 3;
    const int u0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);
    Ring ring{&bars, sbase + OFF_RING + (uint32_t)wg * 8192u, 0u, 0u, {0u, 0u, 0u, 0u}, 0u};
    const uint64_t f_img = make_sdesc_sw128(sbase + OFF_F), x0_img = make_sdesc_sw128(sbase + OFF_X0);
    const uint64_t h_img[2] = {make_sdesc_sw128(sbase + OFF_H), make_sdesc_sw128(sbase + OFF_H + IMG)};
    const int nsf = (a.idim + 63) >> 6;
    uint32_t p_f = 0;
    float hreg[2][32];
    float acc[32], g1[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    // element i = 4 jj + 2 h + e of a fragment: unit u0 + 8 h, stream 8 jj + 2 q4 + e
    auto unit_of = [&](int i) { return u0 + 8 * ((i >> 1) & 1); };
    auto stream_of = [&](int i) { return 8 * (i >> 2) + 2 * q4 + (i & 1); };
    // value v of (unit, stream) of fragment element i -> bf16 hi / lo in the image at `img` (K index = unit)
    auto store_img = [&](uint8_t* img, int i, float v) {
      uint16_t hi, lo;
      split1(v, hi, lo);
      const uint32_t off = a_off(stream_of(i), unit_of(i));
      *reinterpret_cast<uint16_t*>(img + off) = hi;
      *reinterpret_cast<uint16_t*>(img + off + SLAB) = lo;
    };
    for (int it = 0; it < my_tiles; ++it) {
      const int b0 = (blockIdx.x + it * gridDim.x) * a.ms;
      const int Mv = min(a.ms, a.B - b0);                    // live streams of the tile (rows Mv.. are never read back)
      // ---- initial hidden state -> fp32 registers + operand images
#pragma unroll
      for (int l = 0; l < 2; ++l) {                          // compile-time l: hreg stays in registers
        if (l >= L) break;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int sm = stream_of(i);
          hreg[l][i] = a.in_cache != nullptr && sm < Mv ? __ldg(a.in_cache + ((size_t)l * a.B + b0 + sm) * H + unit_of(i)) : 0.f;
          store_img(base + OFF_H + l * IMG, i, hreg[l][i]);
        }
      }
      fence_proxy_async();
      owner_barrier();
      const float bp[2] = {__ldg(vec + a.v_bp + u0), __ldg(vec + a.v_bp + u0 + 8)};
      for (int t = 0; t < T; ++t) {
        // ================= x0 = relu(Linear + b)  -> X0 image                     (subsampling.py:53-57)
        wait_flip(&bars.f_rdy, p_f);
        for (int s = 0; s < nsf; ++s) {
          const int rem = a.idim - 64 * s;
          ring.slab(acc, f_img + (uint64_t)(s * (2 * SLAB >> 4)), rem >= 64 ? 4 : (rem + 15) >> 4, s == 0);
        }
        ring.finish(acc);
        if (lane == 0) mbar_arrive(&bars.lin_bar);          // the feature image may be rewritten
#pragma unroll
        for (int i = 0; i < 32; ++i) store_img(base + OFF_X0, i, fmaxf(acc[i] + bp[(i >> 1) & 1], 0.f));
        fence_proxy_async();
        owner_barrier();
        // ================= GRU layers: x = x0 (layer 0) or the new h of layer 0 (layer 1)
#pragma unroll
        for (int l = 0; l < 2; ++l) {
          if (l >= L) break;
          const float* bih = vec + a.v_layers + (size_t)l * a.v_layer_stride + 2 * H * 3 * H;   // b_ih (384) then b_hh (384)
          const float* bhh = bih + 3 * H;
          float nb_r[2], nb_z[2], b_nx[2], b_nh[2];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int j = u0 + 8 * h;
            nb_r[h] = -LOG2E * (__ldg(bih + j) + __ldg(bhh + j));
            nb_z[h] = -LOG2E * (__ldg(bih + H + j) + __ldg(bhh + H + j));
            b_nx[h] = __ldg(bih + 2 * H + j);
            b_nh[h] = __ldg(bhh + 2 * H + j);
          }
          const uint64_t himg = h_img[l], ximg = l == 0 ? x0_img : h_img[0];
          // r = sigmoid(W_hr h + W_ir x + b)
          ring.gate(acc, himg, true);
          ring.gate(acc, ximg, false);
#pragma unroll
          for (int i = 0; i < 32; ++i) g1[i] = sigmoid_fast(acc[i], nb_r[(i >> 1) & 1]);
          // r * (W_hn h + b_hn)
          ring.gate(acc, himg, true);
#pragma unroll
          for (int i = 0; i < 32; ++i) g1[i] *= acc[i] + b_nh[(i >> 1) & 1];
          // n = tanh(W_in x + b_in + r * (W_hn h + b_hn))
          ring.gate(acc, ximg, true);
#pragma unroll
          for (int i = 0; i < 32; ++i) g1[i] = tanh_fast(acc[i] + b_nx[(i >> 1) & 1] + g1[i]);
          // z = sigmoid(W_hz h + W_iz x + b); h' = (1 - z) n + z h
          ring.gate(acc, himg, true);
          ring.gate(acc, ximg, false);
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const float z = sigmoid_fast(acc[i], nb_z[(i >> 1) & 1]);
            hreg[l][i] = g1[i] + z * (hreg[l][i] - g1[i]);
          }
          owner_barrier();                                   // every warpgroup's GEMMs have read the old h image
#pragma unroll
          for (int i = 0; i < 32; ++i) store_img(base + OFF_H + l * IMG, i, hreg[l][i]);
          fence_proxy_async();
          owner_barrier();
        }
        // ================= classifier on the top layer's h_t (classifier.py:54-67): one warp per (stream, output)
        {
          // 8 (stream, output) pairs per warp pass: lanes split k, the 8 reductions run interleaved, then lane i finishes
          // pair i (bias, activation, store) -- one latency chain per pass instead of one per pair
          const uint8_t* img = base + OFF_H + (L - 1) * IMG;
          const int npair = Mv * a.odim;
          for (int o0 = 8 * warp; o0 < npair; o0 += 8 * NOW) {
            float cacc[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int o = min(o0 + i, npair - 1);
              const int ms = a.odim == 1 ? o : o / a.odim, jo = a.odim == 1 ? 0 : o - ms * a.odim;
              const float* wc = vec + a.v_wc + jo;             // WcT[k][odim]
              float v = 0.f;
#pragma unroll
              for (int u = 0; u < H / 32; ++u) {
                const int k = lane + 32 * u;
                const uint32_t off = a_off(ms, k);
                const float hv = __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(img + off)) +
                                 __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(img + off + SLAB));
                v = fmaf(__ldg(wc + k * a.odim), hv, v);
              }
              cacc[i] = v;
            }
#pragma unroll
            for (int sft = 16; sft > 0; sft >>= 1)
#pragma unroll
              for (int i = 0; i < 8; ++i) cacc[i] += __shfl_xor_sync(0xffffffffu, cacc[i], sft);
            float mine = cacc[0];
#pragma unroll
            for (int i = 1; i < 8; ++i) mine = lane == i ? cacc[i] : mine;
            const int o = o0 + lane;
            if (lane < 8 && o < npair) {
              const int ms = a.odim == 1 ? o : o / a.odim, jo = a.odim == 1 ? 0 : o - ms * a.odim;
              mine += __ldg(vec + a.v_bc + jo);
              if (a.act == WEKWS_ACT_SIGMOID) mine = sigmoidf_acc(mine);
              a.out[((size_t)(b0 + ms) * T + t) * a.odim + jo] = mine;
            }
          }
        }
      }
      // ---- final hidden state
#pragma unroll
      for (int l = 0; l < 2; ++l) {
        if (l >= L) break;
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int sm = stream_of(i);
          if (sm < Mv) a.out_cache[((size_t)l * a.B + b0 + sm) * H + unit_of(i)] = hreg[l][i];
        }
      }
      // the top layer's image is rewritten by the next tile's prologue: every owner must be done with its classifier
      // reads
      owner_barrier();
    }
  }
}

}  // namespace

size_t gru_tc_image_bytes(int L, int idim) { return (size_t)(2 * ((idim + 63) / 64) + 24 * L) * CHUNK; }

bool gru_tc_eligible(int L, int H_, int idim) { return H_ == H && (L == 1 || L == 2) && idim >= 1 && idim <= 96; }

// host: the per-step weight stream, in the order the MMA issuer consumes it.  Every chunk is a K-major SWIZZLE_128B
// bf16 image of 128 rows (hidden units) x 64 K (tc_common.cuh layout: row n at n*128, 16-byte chunk c of the slab at
// chunk c ^ (n & 7)); per K slab a hi chunk then a lo chunk.  Order: Linear; per layer the gates in the order the
// kernel computes them: r (W_hr, W_ir), n (W_hn, then W_in), z (W_hz, W_iz).
void gru_tc_pack(uint8_t* dst, const float* wp /*[H][idim]*/, int idim, const float* const* wih /*[L] of [3H][H]*/,
                 const float* const* whh, int L) {
  uint8_t* p = dst;
  auto slab = [&](const float* W, int ld, int row0, int k0, int kn) {    // rows row0..row0+127, K k0..k0+kn-1
    tc::write_sw128_bf16x3(p, H, W + (size_t)row0 * ld + k0, ld, 1, H, kn);
    p += 2 * CHUNK;
  };
  for (int s = 0; s * 64 < idim; ++s) slab(wp, idim, 0, 64 * s, idim - 64 * s < 64 ? idim - 64 * s : 64);
  auto gate = [&](const float* W, int g) {
    for (int s = 0; s < 2; ++s) slab(W, H, g * H, 64 * s, 64);
  };
  for (int l = 0; l < L; ++l) {
    gate(whh[l], 0); gate(wih[l], 0);        // r
    gate(whh[l], 2);                         // n, h part
    gate(wih[l], 2);                         // n, x part
    gate(whh[l], 1); gate(wih[l], 1);        // z
  }
}

int gru_tc_launch(GruTcArgs a, cudaStream_t st) {
  WEKWS_REQUIRE(a.B >= 1 && a.T >= 1, "gru_tc_launch: empty call");
  // streams per tile: fewer streams per CTA shorten the gate math on the critical path of a step (it is SFU-bound: six
  // ex2 / rcp per unit and stream), the weight stream per CTA and step is the same 786 KB whatever the tile holds
  const int sms0 = device_sm_count();
  a.ms = a.B > 32 * sms0 ? 64 : a.B > 16 * sms0 ? 32 : 16;
  a.n_tiles = (a.B + a.ms - 1) / a.ms;
  if (const int rc = opt_in_smem((const void*)gru_tc_kernel, SMEM_BYTES)) return rc;
  const int sms = device_sm_count();
  const int grid = a.n_tiles < sms ? a.n_tiles : sms;
  gru_tc_kernel<<<grid, NT, SMEM_BYTES, st>>>(a);
  return check_launch("gru_tc_kernel");
}

}  // namespace wekws
