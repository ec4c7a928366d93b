// Per-frame core of the Kaldi-compatible Fbank front-end (fbank.cu): DC removal, pre-emphasis with replicate padding,
// window, 512-point real FFT as a 256-point complex FFT (radix 8 / 8 / 4 Stockham, first radix-8 in registers, two
// exchanges through ONE padded per-warp shared buffer, last pass left in registers), untangle by warp shuffles + power
// spectrum.  One warp per frame.  torchaudio kaldi.py:183-211, 616-618.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dither.cuh"

namespace wekws {
namespace fbcore {

constexpr int WIN = 400, SHIFT = 160, NFFT = 512, NBIN = 256;
constexpr int E_SZ = 280;                   // padded exchange buffer of a warp (complex elements)

// 8-byte (re, im) elements: a half-warp is served in one pass when its 16 elements fall into 16 different 8-byte bank
// pairs (element index mod 16).  First exchange: element i at i + i / 16 (write 8 lane + k -> 8 lane + lane / 2 + k,
// read lane + 32 r -> lane + lane / 16 + 34 r); second exchange: element i at i + 8 (i / 64) (write q + 64 p + 8 k ->
// q + 72 p + 8 k, read q' + 64 r -> q' + 72 r).  All four patterns are conflict-free (checked exhaustively).

__device__ __forceinline__ void cmul(float& re, float& im, float wr, float wi) {
  const float t = re * wr - im * wi;
  im = fmaf(re, wi, im * wr);
  re = t;
}

// In-place 8-point DFT (forward, e^{-2 pi i rk/8}) of (r[], i[]).
__device__ __forceinline__ void dft8(float (&r)[8], float (&i)[8]) {
  const float b0r = r[0] + r[4], b0i = i[0] + i[4], b1r = r[0] - r[4], b1i = i[0] - i[4];
  const float b2r = r[2] + r[6], b2i = i[2] + i[6], b3r = r[2] - r[6], b3i = i[2] - i[6];
  const float b4r = r[1] + r[5], b4i = i[1] + i[5], b5r = r[1] - r[5], b5i = i[1] - i[5];
  const float b6r = r[3] + r[7], b6i = i[3] + i[7], b7r = r[3] - r[7], b7i = i[3] - i[7];
  // c1 = b1 - i b3, c3 = b1 + i b3   (-i (x+iy) = y - ix)
  const float c0r = b0r + b2r, c0i = b0i + b2i, c2r = b0r - b2r, c2i = b0i - b2i;
  const float c1r = b1r + b3i, c1i = b1i - b3r, c3r = b1r - b3i, c3i = b1i + b3r;
  const float c4r = b4r + b6r, c4i = b4i + b6i, c6r = b4r - b6r, c6i = b4i - b6i;
  const float c5r = b5r + b7i, c5i = b5i - b7r, c7r = b5r - b7i, c7i = b5i + b7r;
  const float h = 0.70710678118654752440f;
  // w1*c5, w1 = (1 - i)/sqrt2 ; w3*c7, w3 = (-1 - i)/sqrt2
  const float t5r = h * (c5r + c5i), t5i = h * (c5i - c5r);
  const float t7r = h * (c7i - c7r), t7i = -h * (c7r + c7i);
  r[0] = c0r + c4r; i[0] = c0i + c4i; r[4] = c0r - c4r; i[4] = c0i - c4i;
  r[1] = c1r + t5r; i[1] = c1i + t5i; r[5] = c1r - t5r; i[5] = c1i - t5i;
  r[2] = c2r + c6i; i[2] = c2i - c6r; r[6] = c2r - c6i; i[6] = c2i + c6r;   // -i c6
  r[3] = c3r + t7r; i[3] = c3i + t7i; r[7] = c3r - t7r; i[7] = c3i - t7i;
}


// lane-constant twiddles: pass 1 W_256^(lane k), pass 2 W_32^(p k) = W_256^(8 p k), p = lane / 8
struct LaneTwiddles {
  float t1r[8], t1i[8], t2r[8], t2i[8];
  __device__ __forceinline__ void load(const float2* __restrict__ tw256, int lane) {
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      const float2 w1 = tw256[lane * k];
      const float2 w2 = tw256[8 * (lane >> 3) * k];
      t1r[k] = w1.x; t1i[k] = w1.y; t2r[k] = w2.x; t2i[k] = w2.y;
    }
  }
};

// Power spectrum of one frame -> pw[0..255].  s: the frame's 400 samples as float (int16 scale).  E: E_SZ complex
// elements private to the warp (both exchanges go through it as 8-byte loads / stores; pw may alias it).  s_win: window
// as (even, odd) pairs; s_tw512h: 0.5 W_512^k, k < 256 (the 1/2 of the real-FFT untangle folded into the table: an exact
// scaling, so the result is bit-identical to 0.5 (a +- b) followed by the rotation).  All 32 lanes participate.
// After the last radix-4 pass lane l holds Z[l + 32 i], i < 8, in registers; the untangle needs Z[256 - k]
// next to Z[k], which is element 7 - i of lane 32 - l (lane 0: its own element (8 - i) & 7) -- 16 shuffles instead
// of a third trip through shared memory.
//
// DITHER (training front-end, dither.cuh): the frame's samples get dither * normal_pair(key, b, f, m) in registers as
// they are read; the staged PCM, which overlapping frames share, stays undithered.  The DC mean is then taken over the
// dithered frame, and pre-emphasis needs the dithered sample 2m - 1: it is the odd sample of point m - 1, so it is
// shuffled over from the lane that owns that point (lane 31 of the previous step for lane 0) rather than recomputed,
// which would cost lane 0 a second Philox call and Box-Muller pair per step with the other 31 lanes idle.  Both lanes
// then use the same float, as the reference's single dithered frame does.
template <bool DITHER = false>
__device__ __forceinline__ void frame_power_spectrum(const float* __restrict__ s, const float2* __restrict__ s_win,
                                                     const float2* __restrict__ s_tw512h, const LaneTwiddles& tw, float2* E,
                                                     float* pw, float preemph, int remove_dc, int lane,
                                                     float dither = 0.f, uint32_t key0 = 0, uint32_t key1 = 0,
                                                     int row = 0, int frame = 0) {
  const float* t1r = tw.t1r; const float* t1i = tw.t1i; const float* t2r = tw.t2r; const float* t2i = tw.t2i;
  // ---- window: lane owns packed points m = lane + 32 i (even/odd sample pair 2m, 2m+1) ----
  float xa[7], xb[7], xc[7];
  float sum = 0.f;
  if constexpr (DITHER) {
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      const int m = lane + 32 * i;
      if (m < WIN / 2) {
        const float2 v = *reinterpret_cast<const float2*>(s + 2 * m);
        const float2 n = dither::normal_pair(key0, key1, row, frame, m);
        xb[i] = __fadd_rn(v.x, __fmul_rn(n.x, dither));
        xc[i] = __fadd_rn(v.y, __fmul_rn(n.y, dither));
        sum += xb[i] + xc[i];
      } else {
        xb[i] = xc[i] = 0.f;
      }
    }
#pragma unroll
    for (int i = 0; i < 7; ++i) {
      const float up = __shfl_up_sync(0xffffffffu, xc[i], 1);
      const float wrap = i > 0 ? __shfl_sync(0xffffffffu, xc[i > 0 ? i - 1 : 0], 31) : xb[0];
      xa[i] = lane > 0 ? up : wrap;                   // point 0: replicate pad of the dithered x[0] (kaldi.py:195)
    }
  } else {
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const int m = lane + 32 * i;
    if (m < WIN / 2) {
      const float2 v = *reinterpret_cast<const float2*>(s + 2 * m);
      xb[i] = v.x; xc[i] = v.y;
      xa[i] = m > 0 ? s[2 * m - 1] : xb[i];           // replicate pad (kaldi.py:195)
      sum += xb[i] + xc[i];
    } else {
      xa[i] = xb[i] = xc[i] = 0.f;
    }
  }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = remove_dc ? sum * (1.0f / (float)WIN) : 0.f;   // (the reference's torch.mean sums in another order anyway)
  float zr[8], zi[8];
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const int m = lane + 32 * i;
    if (m < WIN / 2) {
      const float2 w = s_win[m];
      const float pa = xa[i] - mean, pb = xb[i] - mean, pc = xc[i] - mean;
      zr[i] = (pb - preemph * pa) * w.x;
      zi[i] = (pc - preemph * pb) * w.y;
    } else {
      zr[i] = 0.f; zi[i] = 0.f;
    }
  }
  zr[7] = 0.f; zi[7] = 0.f;

  // ---- pass 1: radix 8 over r (n=256, s=1) -> E[8p + k] * W_256^(pk) ----
  dft8(zr, zi);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (k) cmul(zr[k], zi[k], t1r[k], t1i[k]);
    E[8 * lane + (lane >> 1) + k] = make_float2(zr[k], zi[k]);
  }
  __syncwarp();
  // ---- pass 2: radix 8 (n=32, s=8): j = q + 8p reads E[j + 32r], writes E'[q + 64p + 8k] ----
  {
    const int b = lane + (lane >> 4);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      const float2 v = E[b + 34 * r];
      zr[r] = v.x; zi[r] = v.y;
    }
  }
  __syncwarp();                                   // same buffer, other layout: every lane has read before any writes
  dft8(zr, zi);
  {
    const int b = (lane & 7) + 72 * (lane >> 3);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if (k) cmul(zr[k], zi[k], t2r[k], t2i[k]);
      E[b + 8 * k] = make_float2(zr[k], zi[k]);
    }
  }
  __syncwarp();
  // ---- pass 3: radix 4 (n=4, s=64): q = lane + 32 hh reads E'[q + 64r]; Z[q + 64k] stays in registers as element hh + 2k
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const int q = lane + 32 * hh;
    const float2 v0 = E[q], v1 = E[q + 72], v2 = E[q + 144], v3 = E[q + 216];
    const float s0r = v0.x + v2.x, s0i = v0.y + v2.y, d0r = v0.x - v2.x, d0i = v0.y - v2.y;
    const float s1r = v1.x + v3.x, s1i = v1.y + v3.y, d1r = v1.x - v3.x, d1i = v1.y - v3.y;
    zr[hh] = s0r + s1r;      zi[hh] = s0i + s1i;
    zr[hh + 2] = d0r + d1i;  zi[hh + 2] = d0i - d1r;     // d0 - i d1
    zr[hh + 4] = s0r - s1r;  zi[hh + 4] = s0i - s1i;
    zr[hh + 6] = d0r - d1i;  zi[hh + 6] = d0i + d1r;     // d0 + i d1
  }
  __syncwarp();                                   // the exchange buffer is free again (pw may alias it)
  // ---- real-FFT untangle + power spectrum -> pw[0..255] ----
  float cr[8], ci[8];
  {
    const int src = (32 - lane) & 31;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      cr[j] = __shfl_sync(0xffffffffu, zr[j], src);
      ci[j] = __shfl_sync(0xffffffffu, zi[j], src);
    }
  }
  const bool l0 = lane == 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = lane + 32 * i;
    const float ar = zr[i], ai = zi[i];
    const float pr = l0 ? cr[(8 - i) & 7] : cr[7 - i], pi = l0 ? ci[(8 - i) & 7] : ci[7 - i];
    const float sr = ar + pr, si = ai - pi, dr = ar - pr, di = ai + pi;
    const float2 w = s_tw512h[k];
    const float p = w.x * dr - w.y * di, q = w.x * di + w.y * dr;
    const float xr = fmaf(0.5f, sr, q), xi = fmaf(0.5f, si, -p);
    pw[k] = xr * xr + xi * xi;
  }
  __syncwarp();
}

}  // namespace fbcore
}  // namespace wekws
