// Training-audio augmentation of the legacy data chain (wekws/dataset/processor.py add_reverb / add_noise) for a
// batch of rows.  The host draws which rows are augmented and with which clip (Python's `random`, the reference's
// order) and uploads only the selected clips; these kernels do the arithmetic.
//
// Reverb: y[i] = sum_{k <= min(i, L - 1)} h[k] x[i - k] for i < n (convolve(x, h, 'full')[:n]), h = rir / sqrt(sum
// rir^2).  One CTA per (row, tile of kRvTile outputs).  The CTA forms sum rir^2 over all L taps in double in a fixed
// order, then walks the taps k < min(L, n, tile end) in chunks: each chunk's taps and the matching input window are
// staged in shared memory as doubles, and each thread keeps kRvPer consecutive outputs and the kRvPer input samples
// they need in registers, sliding the samples by one register per tap.  Per tap a thread issues one window load, a
// broadcast tap load (two taps per 16-byte load) and kRvPer FP64 FMAs; the window is stored with one pad double per
// kRvPer so that the lanes' loads (kRvPer + 1 doubles apart) hit distinct banks.  Products of float32 samples and
// float32 taps are exact in double, the sum is rounded in double only, and the output is acc / sqrt(sum rir^2)
// rounded once to float32: within 1 ulp of the float64 evaluation.
//
// Noise: one CTA per row.  audio_db = 10 log10(mean((x 2^-15)^2) + 1e-4) (the reference's waveform is at [-1, 1]
// scale here, ours at int16 scale), noise_db = 10 log10(mean(s^2) + 1e-4) over the segment used, each mean summed in
// double in a fixed order; gain = 2^15 sqrt(10^((audio_db - noise_db - snr) / 10)) = 2^15 10^((...) / 20) in double, rounded once; then
// y[i] = x[i] + gain s[i] as one float32 multiply and one float32 add, the reference's two roundings at 2^15 times
// its scale (exact: a power of two).
#include <stdint.h>

#include "common.cuh"

namespace wekws {
namespace {

constexpr int kRvThreads = 256;
constexpr int kRvPer = 8;                              // consecutive outputs per thread
constexpr int kRvTile = kRvThreads * kRvPer;           // outputs per CTA
constexpr int kRvChunk = 512;                          // taps staged per step
constexpr int kRvWin = kRvTile + kRvChunk;             // staged input samples per step (one spare)
constexpr int kRvWinPad = kRvWin + kRvWin / kRvPer;    // with one pad double per kRvPer
constexpr int kNzThreads = 256;

__device__ __forceinline__ double to_double(float v) { return (double)v; }
__device__ __forceinline__ double to_double(int16_t v) { return (double)v; }
__device__ __forceinline__ int pad_index(int w) { return w + w / kRvPer; }

// sum of v over the CTA in a fixed order (lane tree, then the warps in order); every thread gets the result
__device__ double block_sum(double v, double* s_red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();                                     // s_red is free
  if ((threadIdx.x & 31) == 0) s_red[warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int w = 0; w < nw; ++w) t += s_red[w];
  return t;
}

// rows: (B, 3) int32 (length, offset of the row's RIR in rir, its number of taps; 0 taps = not selected)
template <typename T>
__global__ void __launch_bounds__(kRvThreads) reverb_kernel(const T* __restrict__ pcm, long long pcm_stride,
                                                            long long num_samples, const int32_t* __restrict__ rows,
                                                            const float* __restrict__ rir, float* __restrict__ out,
                                                            long long out_stride) {
  __shared__ __align__(16) double s_h[kRvChunk];
  __shared__ double s_w[kRvWinPad];
  __shared__ double s_red[kRvThreads / 32];
  const long long b = blockIdx.y;
  const long long i0 = (long long)blockIdx.x * kRvTile;
  const long long i1 = i0 + kRvTile < num_samples ? i0 + kRvTile : num_samples;
  const T* x = pcm + b * pcm_stride;
  float* y = out + b * out_stride;
  long long n = __ldg(rows + 3 * b);
  n = n < 0 ? 0 : (n > num_samples ? num_samples : n);
  const int L = __ldg(rows + 3 * b + 2);
  const long long c0 = L > 0 ? (n > i0 ? n : i0) : i0;   // [c0, i1) is a copy of the input
  for (long long i = c0 + threadIdx.x; i < i1; i += kRvThreads) y[i] = (float)x[i];
  if (c0 <= i0) return;                                  // uniform over the CTA
  const float* h = rir + __ldg(rows + 3 * b + 1);
  double ss = 0.0;
  for (int k = threadIdx.x; k < L; k += kRvThreads) {
    const double v = (double)__ldg(h + k);
    ss = fma(v, v, ss);
  }
  const double norm = sqrt(block_sum(ss, s_red));
  const long long iend = c0 < i0 + kRvTile ? c0 : i0 + kRvTile;   // outputs [i0, iend) are convolved
  const long long kmax = (long long)L < iend ? (long long)L : iend;   // taps k <= i < iend
  const int tid = threadIdx.x;
  double acc[kRvPer];
#pragma unroll
  for (int r = 0; r < kRvPer; ++r) acc[r] = 0.0;
  for (long long k0 = 0; k0 < kmax; k0 += kRvChunk) {
    const int kc = (int)(kmax - k0 < kRvChunk ? kmax - k0 : kRvChunk);
    __syncthreads();                                     // the previous chunk is no longer read
    for (int j = tid; j < kRvChunk; j += kRvThreads) s_h[j] = j < kc ? (double)__ldg(h + k0 + j) : 0.0;
    // window sample w is x[g0 + w]; output i0 + 8 tid + r with tap k0 + j reads w = 8 tid + r + kRvChunk - 1 - j
    const long long g0 = i0 - k0 - (kRvChunk - 1);
    for (int w = tid; w < kRvWin; w += kRvThreads) {
      const long long g = g0 + w;
      s_w[pad_index(w)] = (g >= 0 && g < iend) ? to_double(x[g]) : 0.0;
    }
    __syncthreads();
    double xr[kRvPer];
    const int wb = tid * kRvPer + kRvChunk - 1;
#pragma unroll
    for (int r = 0; r < kRvPer; ++r) xr[r] = s_w[pad_index(wb + r)];
    const int ku = (kc + 7) & ~7;
    for (int j = 0; j < ku; j += 8) {
      double hv[8];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const double2 v = reinterpret_cast<const double2*>(s_h + j)[q];
        hv[2 * q] = v.x;
        hv[2 * q + 1] = v.y;
      }
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int r = 0; r < kRvPer; ++r) acc[r] = fma(hv[jj], xr[r], acc[r]);
#pragma unroll
        for (int r = kRvPer - 1; r > 0; --r) xr[r] = xr[r - 1];
        const int w = wb - (j + jj) - 1;                 // -1 only after the last tap of the chunk: never used
        xr[0] = s_w[pad_index(w > 0 ? w : 0)];
      }
    }
  }
  const long long base = i0 + (long long)tid * kRvPer;
#pragma unroll
  for (int r = 0; r < kRvPer; ++r)
    if (base + r < iend) y[base + r] = (float)(acc[r] / norm);
}

// rows: (B, 3) int32 (length, offset of the row's noise segment in noise, its length M; 0 = not selected).  The row
// adds s[i] = noise[offset + i mod M] for i < length: M = length when the clip was longer (the drawn segment), else the
// whole clip, repeated as np.resize does.
template <typename T>
__global__ void __launch_bounds__(kNzThreads) noise_kernel(const T* pcm, long long pcm_stride,
                                                           long long num_samples, const int32_t* __restrict__ rows,
                                                           const double* __restrict__ snr,
                                                           const float* __restrict__ noise, float* out,
                                                           long long out_stride, bool in_place) {
  __shared__ double s_red[kNzThreads / 32];
  const long long b = blockIdx.x;
  const T* x = pcm + b * pcm_stride;
  float* y = out + b * out_stride;
  long long n = __ldg(rows + 3 * b);
  n = n < 0 ? 0 : (n > num_samples ? num_samples : n);
  const int M = __ldg(rows + 3 * b + 2);
  const long long c0 = M > 0 ? n : 0;                    // [c0, num_samples) is a copy of the input
  if (!in_place)
    for (long long i = c0 + threadIdx.x; i < num_samples; i += kNzThreads) y[i] = (float)x[i];
  if (c0 == 0) return;                                   // uniform over the CTA
  const float* s = noise + __ldg(rows + 3 * b + 1);
  double sa = 0.0, sn = 0.0;
  const unsigned un = (unsigned)n, um = (unsigned)M;    // n < 2^31 (checked on the host)
  for (unsigned i = threadIdx.x; i < un; i += kNzThreads) {
    const double a = to_double(x[i]) * 0x1p-15;
    const double v = (double)s[i % um];
    sa = fma(a, a, sa);
    sn = fma(v, v, sn);
  }
  sa = block_sum(sa, s_red);
  sn = block_sum(sn, s_red);
  const double audio_db = 10.0 * log10(sa / (double)n + 1e-4);
  const double noise_db = 10.0 * log10(sn / (double)n + 1e-4);
  const float gain = (float)(32768.0 * exp10((audio_db - noise_db - __ldg(snr + b)) / 20.0));   // sqrt(10^(d/10))
  for (unsigned i = threadIdx.x; i < un; i += kNzThreads)
    y[i] = __fadd_rn((float)x[i], __fmul_rn(gain, s[i % um]));
}

}  // namespace
}  // namespace wekws

using namespace wekws;

extern "C" int wekws_reverb(const void* d_pcm, int pcm_dtype, int64_t B, int64_t num_samples, int64_t pcm_stride,
                            const int32_t* d_rows, const float* d_rir, float* d_out, int64_t out_stride,
                            void* stream) {
  WEKWS_REQUIRE(B >= 0 && num_samples >= 0, "wekws_reverb: negative size");
  WEKWS_REQUIRE(pcm_dtype == WEKWS_PCM_S16 || pcm_dtype == WEKWS_PCM_F32, "wekws_reverb: bad pcm_dtype %d", pcm_dtype);
  WEKWS_REQUIRE(B <= 1 || (pcm_stride >= num_samples && out_stride >= num_samples),
                "wekws_reverb: a row stride is shorter than its row");
  WEKWS_REQUIRE(B <= 65535, "wekws_reverb: %lld rows, more than one launch takes (65535)", (long long)B);
  if (B == 0 || num_samples == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_pcm && d_rows && d_rir && d_out, "wekws_reverb: null pointer");
  WEKWS_REQUIRE(d_pcm != (const void*)d_out, "wekws_reverb: the output must be a separate buffer");
  const dim3 grid((unsigned)((num_samples + kRvTile - 1) / kRvTile), (unsigned)B);
  cudaStream_t st = (cudaStream_t)stream;
  if (pcm_dtype == WEKWS_PCM_S16)
    reverb_kernel<int16_t><<<grid, kRvThreads, 0, st>>>(static_cast<const int16_t*>(d_pcm), pcm_stride, num_samples,
                                                        d_rows, d_rir, d_out, out_stride);
  else
    reverb_kernel<float><<<grid, kRvThreads, 0, st>>>(static_cast<const float*>(d_pcm), pcm_stride, num_samples,
                                                      d_rows, d_rir, d_out, out_stride);
  return check_launch("reverb_kernel");
}

extern "C" int wekws_add_noise(const void* d_pcm, int pcm_dtype, int64_t B, int64_t num_samples, int64_t pcm_stride,
                               const int32_t* d_rows, const double* d_snr, const float* d_noise, float* d_out,
                               int64_t out_stride, void* stream) {
  WEKWS_REQUIRE(B >= 0 && num_samples >= 0, "wekws_add_noise: negative size");
  WEKWS_REQUIRE(pcm_dtype == WEKWS_PCM_S16 || pcm_dtype == WEKWS_PCM_F32, "wekws_add_noise: bad pcm_dtype %d",
                pcm_dtype);
  WEKWS_REQUIRE(B <= 1 || (pcm_stride >= num_samples && out_stride >= num_samples),
                "wekws_add_noise: a row stride is shorter than its row");
  if (B == 0 || num_samples == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_pcm && d_rows && d_snr && d_noise && d_out, "wekws_add_noise: null pointer");
  const bool in_place = d_pcm == (const void*)d_out;
  WEKWS_REQUIRE(!in_place || (pcm_dtype == WEKWS_PCM_F32 && pcm_stride == out_stride),
                "wekws_add_noise: in place needs float32 input with the output's row stride");
  WEKWS_REQUIRE(B < (1ll << 31) && num_samples < (1ll << 31), "wekws_add_noise: %lld x %lld samples is out of range",
                (long long)B, (long long)num_samples);
  cudaStream_t st = (cudaStream_t)stream;
  if (pcm_dtype == WEKWS_PCM_S16)
    noise_kernel<int16_t><<<(unsigned)B, kNzThreads, 0, st>>>(static_cast<const int16_t*>(d_pcm), pcm_stride,
                                                              num_samples, d_rows, d_snr, d_noise, d_out, out_stride,
                                                              in_place);
  else
    noise_kernel<float><<<(unsigned)B, kNzThreads, 0, st>>>(static_cast<const float*>(d_pcm), pcm_stride,
                                                            num_samples, d_rows, d_snr, d_noise, d_out, out_stride,
                                                            in_place);
  return check_launch("noise_kernel");
}
