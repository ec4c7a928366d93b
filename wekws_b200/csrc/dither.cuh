// Gaussian dither noise of the training front-end (torchaudio kaldi.py `_get_window`: strided_input +
// torch.randn(m, frame_length) * dither, added to the framed signal before DC removal, pre-emphasis and the window).
//
// No device generator reproduces torch's CPU randn, so the noise is a pure, documented function of
// (seed, row b, frame f, sample j), j < 400, that the tests restate in float64 (oracle/kws_train_oracle.py):
//   words = Philox4x32-10(counter = (j / 4, f, b, 0), key = (seed lo, seed hi)), Random123 constants;
//   u_i   = ((words_i >> 8) + 0.5) 2^-24, in (0, 1), never 0;
//   samples 4q, 4q+1 = r (cos 2 pi u_1, sin 2 pi u_1), r = sqrt(-2 ln u_0)    (first Box-Muller pair)
//   samples 4q+2, 4q+3 = the same with (u_2, u_3)                               (second pair).
// Evaluation in float32: with u = n 2^-25 (n odd, < 2^25), u itself is exact only for n < 2^24, so the top half
// takes ln u = log1p(-(2^25 - n) 2^-25) (exact argument; ln(1 - t) for tiny t would otherwise cancel) and the bottom
// half MUFU lg2 + one Newton step with a split ln 2; 2 u is reduced to (-1, 1] by its period before sincospif, again
// an exact argument.  Against the float64 formula each normal is within 1e-6 absolute (tests/test_train_features.py
// bounds it; |normal| <= 5.9).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace wekws {
namespace dither {

constexpr uint32_t PHILOX_M0 = 0xD2511F53u, PHILOX_M1 = 0xCD9E8D57u;
constexpr uint32_t PHILOX_W0 = 0x9E3779B9u, PHILOX_W1 = 0xBB67AE85u;

__host__ __device__ __forceinline__ uint32_t mulhi32(uint32_t a, uint32_t b) {
#ifdef __CUDA_ARCH__
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * b) >> 32);
#endif
}

__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += PHILOX_W0; k1 += PHILOX_W1; }
    const uint32_t lo0 = PHILOX_M0 * c.x, hi0 = mulhi32(PHILOX_M0, c.x);
    const uint32_t lo1 = PHILOX_M1 * c.z, hi1 = mulhi32(PHILOX_M1, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// ln u for u = n 2^-25, n odd (the u of a word w is n = 2 (w >> 8) + 1)
__device__ __forceinline__ float ln_uniform(uint32_t n) {
  if (n >= (1u << 24)) return log1pf(-__uint2float_rn((1u << 25) - n) * 0x1p-25f);
  const float x = __uint2float_rn(n) * 0x1p-25f;             // exact
  float t, e;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-t));
  // ln x = ln2 t + ln(x 2^-t), |x 2^-t - 1| < 1e-6; ln 2 split so that ln2 t carries no rounding of the constant
  return __fmaf_rn(0.693145751953125f, t, __fmaf_rn(1.42860682030941723212e-6f, t, __fmaf_rn(x, e, -1.0f)));
}

// One Box-Muller pair from the words (wa, wb): (r cos 2 pi u_b, r sin 2 pi u_b), r = sqrt(-2 ln u_a)
__device__ __forceinline__ float2 box_muller(uint32_t wa, uint32_t wb) {
  const float r = __fsqrt_rn(-2.0f * ln_uniform(2u * (wa >> 8) + 1u));
  const uint32_t nb = 2u * (wb >> 8) + 1u;                    // 2 u_b = nb 2^-24, reduced to (-1, 1]
  const float y = nb < (1u << 24) ? __uint2float_rn(nb) * 0x1p-24f : -__uint2float_rn((1u << 25) - nb) * 0x1p-24f;
  float s, c;
  sincospif(y, &s, &c);
  return make_float2(__fmul_rn(r, c), __fmul_rn(r, s));
}

// The two normals of sample pair p (samples 2p, 2p + 1) of frame f of row b
__device__ __forceinline__ float2 normal_pair(uint32_t k0, uint32_t k1, int b, int f, int p) {
  const uint4 w = philox4x32_10(make_uint4((uint32_t)p >> 1, (uint32_t)f, (uint32_t)b, 0u), k0, k1);
  return (p & 1) ? box_muller(w.z, w.w) : box_muller(w.x, w.y);
}

}  // namespace dither
}  // namespace wekws
