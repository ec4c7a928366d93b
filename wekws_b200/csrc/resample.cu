// torchaudio.transforms.Resample(orig_freq, new_freq) (sinc_interp_hann, lowpass_filter_width 6, rolloff 0.99; the
// resampling of wekws/dataset/processor.py resample() and tools/compute_cmvn_stats.py) for a batch of waveforms.
//
// torchaudio 2.11 _apply_sinc_resample_kernel: with O = orig / gcd and N = new / gcd, pad the waveform with `width`
// zeros on the left and width + O on the right, run conv1d with the (N, 2 width + O) kernel at stride O, interleave
// the N phases and keep ceil(N len / O) outputs.  So output j = n N + p (phase p of frame n) is
//     y[j] = sum_k kernel[p][k] * x[n O + k - width],   x = 0 outside [0, len).
// The Hann window clamps the sinc outside +-6 zero crossings, so most of the dense table is exact zeros: the handle
// keeps each phase's span from its first to its last non-zero tap only, and the kernel never reads a zero.
//
// One persistent CTA loads that compact table into shared memory once, as doubles, then walks (row, tile) items: a
// tile is F frames of N outputs; the CTA stages the tile's input window ((F - 1) O + 2 width + O samples, zeros
// outside the row) in shared memory as doubles, with 16-byte loads where the row is aligned, and each thread forms its
// outputs with FP64 FMAs (a float32 x float32 product is exact in double) and rounds once to float32.  Every tap and
// every input sample is converted to double once per CTA or tile, not once per product.  Samples at or past lens[b]
// are replaced by zeros, never read as data; outputs past a row's length are written as zeros.
#include <stdint.h>

#include <new>
#include <vector>

#include "common.cuh"

namespace wekws {
namespace {

constexpr int kRsThreads = 256;
constexpr int kRsTileOutputs = 2048;        // outputs per tile (at least one frame of N)
constexpr int kRsWindowMax = 8192;          // staged input samples per tile, as doubles: 64 KB
constexpr int kRsTableMax = 96 * 1024;      // bytes of compact taps (doubles) + per-phase offsets in shared memory

// torchaudio's target length: ceil(torch.as_tensor(N * len / O)), i.e. the double quotient rounded to float32 before
// the ceil (so past about 2^24 / O outputs it can drop the last partial sample), and never past the conv1d's
// (len / O + 1) N outputs
__host__ __device__ __forceinline__ long long rs_out_len(long long len, long long O, long long N) {
  if (len <= 0) return 0;
  const float q = (float)((double)(N * len) / (double)O);
  const long long t = (long long)ceilf(q), conv = (len / O + 1) * N;
  return t < conv ? t : conv;
}

__device__ __forceinline__ double to_double(float v) { return (double)v; }
__device__ __forceinline__ double to_double(int16_t v) { return (double)v; }

// s_win[i] = x[g0 + i] for 0 <= g0 + i < len, 0 otherwise, i in [0, win)
template <typename T>
__device__ __forceinline__ void stage_window(const T* __restrict__ row, long long g0, long long len, int win,
                                             bool vec_ok, double* __restrict__ s_win) {
  constexpr int V = 16 / sizeof(T);
  if (!vec_ok) {
    for (int i = threadIdx.x; i < win; i += blockDim.x) {
      const long long gi = g0 + i;
      s_win[i] = (gi >= 0 && gi < len) ? to_double(row[gi]) : 0.0;
    }
    return;
  }
  const long long a0 = g0 >= 0 ? g0 / V * V : -((-g0 + V - 1) / V) * V;
  const long long a1 = g0 + win;
  for (long long c = a0 + (long long)threadIdx.x * V; c < a1; c += (long long)blockDim.x * V) {
    T v[V];
    if (c >= 0 && c + V <= len) {
      *reinterpret_cast<int4*>(v) = __ldg(reinterpret_cast<const int4*>(row + c));
    } else {
#pragma unroll
      for (int e = 0; e < V; ++e) v[e] = (c + e >= 0 && c + e < len) ? row[c + e] : T(0);
    }
#pragma unroll
    for (int e = 0; e < V; ++e) {
      const long long i = c + e - g0;
      if (i >= 0 && i < win) s_win[i] = to_double(v[e]);
    }
  }
}

struct ResampleArgs {
  const void* pcm;
  long long pcm_stride, num_samples, B;
  const int32_t* lens;
  float* out;
  long long out_stride, max_out, tiles_per_row;
  const float* taps;
  const int* off;      // (N + 1): phase p's taps are taps[off[p] .. off[p + 1])
  const int* first;    // (N): the kernel column of phase p's first kept tap
  int O, N, width, F, win, ntaps, win_off;   // win_off: byte offset of the window in shared memory
  bool vec_ok;
};

template <typename T>
__global__ void __launch_bounds__(kRsThreads) resample_kernel(const ResampleArgs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  double* s_taps = reinterpret_cast<double*>(smem);
  int* s_off = reinterpret_cast<int*>(s_taps + a.ntaps);
  int* s_first = s_off + a.N + 1;
  double* s_win = reinterpret_cast<double*>(smem + a.win_off);
  for (int i = threadIdx.x; i < a.ntaps; i += blockDim.x) s_taps[i] = (double)a.taps[i];
  for (int i = threadIdx.x; i <= a.N; i += blockDim.x) s_off[i] = a.off[i];
  for (int i = threadIdx.x; i < a.N; i += blockDim.x) s_first[i] = a.first[i];
  const long long tile_out = (long long)a.F * a.N;
  const long long items = a.B * a.tiles_per_row;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const long long b = it / a.tiles_per_row, tile = it - b * a.tiles_per_row;
    long long len = a.lens ? (long long)a.lens[b] : a.num_samples;
    len = len < 0 ? 0 : (len > a.num_samples ? a.num_samples : len);
    const long long out_len = rs_out_len(len, a.O, a.N);
    const long long j0 = tile * tile_out;
    const long long j1 = j0 + tile_out < a.max_out ? j0 + tile_out : a.max_out;
    float* orow = a.out + b * a.out_stride;
    if (j0 >= out_len) {                       // the whole tile is padding (uniform over the CTA)
      for (long long j = j0 + threadIdx.x; j < j1; j += blockDim.x) orow[j] = 0.f;
      continue;
    }
    const long long n0 = tile * a.F;
    __syncthreads();                           // the table is loaded / the previous tile's window is no longer read
    stage_window<T>(static_cast<const T*>(a.pcm) + b * a.pcm_stride, n0 * a.O - a.width, len, a.win, a.vec_ok, s_win);
    __syncthreads();
    const int nj = (int)(j1 - j0);
    for (int jl = threadIdx.x; jl < nj; jl += blockDim.x) {
      float y = 0.f;
      if (j0 + jl < out_len) {
        const int nl = jl / a.N, p = jl - nl * a.N;
        const int o = s_off[p], c = s_off[p + 1] - o;
        const double* w = s_win + nl * a.O + s_first[p];
        const double* tp = s_taps + o;
        double acc = 0.0;
        for (int i = 0; i < c; ++i) acc = fma(tp[i], w[i], acc);
        y = (float)acc;
      }
      orow[j0 + jl] = y;
    }
  }
}

long long gcd_ll(long long a, long long b) {
  while (b) { const long long t = a % b; a = b; b = t; }
  return a;
}

}  // namespace
}  // namespace wekws

// ------------------------------------------------------------------------------- C ABI
using namespace wekws;

struct wekws_resample {
  int orig = 0, neu = 0;     // reduced by the gcd
  int width = 0, F = 0, win = 0, ntaps = 0, win_off = 0;
  size_t smem = 0;
  int device = 0;
  int occ[2] = {0, 0};
  float* d_taps = nullptr;
  int* d_off = nullptr;
  int* d_first = nullptr;
};

extern "C" int wekws_resample_create(int orig_freq, int new_freq, const float* h_kernel, int width,
                                     wekws_resample** out) {
  WEKWS_REQUIRE(out, "wekws_resample_create: null output");
  WEKWS_REQUIRE(orig_freq > 0 && new_freq > 0, "resample: rates must be positive (got %d -> %d)", orig_freq, new_freq);
  WEKWS_REQUIRE(orig_freq != new_freq, "resample: equal rates (%d) need no resampling", orig_freq);
  WEKWS_REQUIRE(h_kernel && width >= 0, "wekws_resample_create: null kernel or negative width");
  const long long g = gcd_ll(orig_freq, new_freq);
  const int O = (int)(orig_freq / g), N = (int)(new_freq / g);
  const long long K = 2ll * width + O;
  WEKWS_REQUIRE(K <= kRsWindowMax, "resample %d -> %d: the filter spans %lld input samples, more than the %d a tile "
                "stages", orig_freq, new_freq, K, kRsWindowMax);
  std::vector<int> off(N + 1), first(N);
  std::vector<float> taps;
  for (int p = 0; p < N; ++p) {
    const float* row = h_kernel + (size_t)p * K;
    long long f = -1, l = -1;
    for (long long k = 0; k < K; ++k)
      if (row[k] != 0.f) { if (f < 0) f = k; l = k; }
    off[p] = (int)taps.size();
    first[p] = f < 0 ? 0 : (int)f;
    if (f >= 0) taps.insert(taps.end(), row + f, row + l + 1);
    const size_t bytes = taps.size() * sizeof(double) + (2 * (size_t)N + 1) * sizeof(int);
    WEKWS_REQUIRE(bytes <= (size_t)kRsTableMax, "resample %d -> %d: the compact filter table needs at least %zu bytes of "
                  "shared memory, more than the %d available to it", orig_freq, new_freq, bytes, kRsTableMax);
  }
  off[N] = (int)taps.size();
  if (taps.empty()) taps.push_back(0.f);
  int F = (kRsTileOutputs + N - 1) / N;
  if ((long long)(F - 1) * O + K > kRsWindowMax) F = (int)((kRsWindowMax - K) / O + 1);
  if (F < 1) F = 1;
  wekws_resample* h = new (std::nothrow) wekws_resample();
  if (!h) { set_error("out of host memory"); return WEKWS_ERR_NOMEM; }
  h->orig = O; h->neu = N; h->width = width; h->F = F;
  h->win = (int)((long long)(F - 1) * O + K);
  h->ntaps = off[N];
  h->win_off = (int)((taps.size() * sizeof(double) + (2 * (size_t)N + 1) * sizeof(int) + 15) & ~(size_t)15);
  h->smem = (size_t)h->win_off + (size_t)h->win * sizeof(double);
  if (cudaGetDevice(&h->device) != cudaSuccess ||
      cudaMalloc((void**)&h->d_taps, taps.size() * sizeof(float)) != cudaSuccess ||
      cudaMalloc((void**)&h->d_off, off.size() * sizeof(int)) != cudaSuccess ||
      cudaMalloc((void**)&h->d_first, first.size() * sizeof(int)) != cudaSuccess ||
      cudaMemcpy(h->d_taps, taps.data(), taps.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(h->d_off, off.data(), off.size() * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(h->d_first, first.data(), first.size() * sizeof(int), cudaMemcpyHostToDevice) != cudaSuccess) {
    const cudaError_t e = cudaGetLastError();
    wekws_resample_destroy(h);
    set_error("wekws_resample_create: %s", cudaGetErrorString(e));
    return WEKWS_ERR_CUDA;
  }
  const void* kern[2] = {(const void*)resample_kernel<int16_t>, (const void*)resample_kernel<float>};
  for (int i = 0; i < 2; ++i) {
    const int rc = opt_in_smem(kern[i], h->smem);     // h->device is current; forward checks it still is
    if (rc != WEKWS_OK) {
      wekws_resample_destroy(h);
      return rc;
    }
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h->occ[i], kern[i], kRsThreads, h->smem) != cudaSuccess) {
      const cudaError_t e = cudaGetLastError();
      wekws_resample_destroy(h);
      set_error("wekws_resample_create: %s", cudaGetErrorString(e));
      return WEKWS_ERR_CUDA;
    }
    if (h->occ[i] < 1) h->occ[i] = 1;
  }
  *out = h;
  return WEKWS_OK;
}

extern "C" void wekws_resample_destroy(wekws_resample* h) {
  if (!h) return;
  cudaFree(h->d_taps); cudaFree(h->d_off); cudaFree(h->d_first);
  delete h;
}

extern "C" int64_t wekws_resample_output_length(const wekws_resample* h, int64_t num_samples) {
  return h ? rs_out_len(num_samples, h->orig, h->neu) : 0;
}

extern "C" int wekws_resample_forward(wekws_resample* h, const void* d_pcm, int pcm_dtype, int64_t B,
                                      int64_t num_samples, int64_t pcm_stride, const int32_t* d_lens, float* d_out,
                                      int64_t out_stride, int64_t max_out, void* stream) {
  WEKWS_REQUIRE(h && d_out, "wekws_resample_forward: null handle or output");
  WEKWS_REQUIRE(B >= 0 && num_samples >= 0 && max_out >= 0, "wekws_resample_forward: negative size");
  WEKWS_REQUIRE(pcm_dtype == WEKWS_PCM_S16 || pcm_dtype == WEKWS_PCM_F32, "wekws_resample_forward: bad pcm_dtype %d",
                pcm_dtype);
  WEKWS_REQUIRE(max_out >= rs_out_len(num_samples, h->orig, h->neu),
                "wekws_resample_forward: max_out %lld < output length of %lld samples (%lld)", (long long)max_out,
                (long long)num_samples, rs_out_len(num_samples, h->orig, h->neu));
  WEKWS_REQUIRE(out_stride >= max_out && (B <= 1 || pcm_stride >= num_samples),
                "wekws_resample_forward: a row stride is shorter than its row");
  WEKWS_REQUIRE(num_samples < (1ll << 40), "wekws_resample_forward: %lld samples per row is out of range",
                (long long)num_samples);
  if (B == 0 || max_out == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_pcm, "wekws_resample_forward: null pcm");
  int dev = 0;
  WEKWS_CUDA_OK(cudaGetDevice(&dev));
  WEKWS_REQUIRE(dev == h->device, "resample handle was created on device %d but the current device is %d", h->device,
                dev);
  const int esz = pcm_dtype == WEKWS_PCM_S16 ? 2 : 4;
  ResampleArgs a;
  a.pcm = d_pcm; a.pcm_stride = pcm_stride; a.num_samples = num_samples; a.B = B; a.lens = d_lens;
  a.out = d_out; a.out_stride = out_stride; a.max_out = max_out;
  const long long tile_out = (long long)h->F * h->neu;
  a.tiles_per_row = (max_out + tile_out - 1) / tile_out;
  a.taps = h->d_taps; a.off = h->d_off; a.first = h->d_first;
  a.O = h->orig; a.N = h->neu; a.width = h->width; a.F = h->F; a.win = h->win; a.ntaps = h->ntaps;
  a.win_off = h->win_off;
  a.vec_ok = (reinterpret_cast<uintptr_t>(d_pcm) & 15) == 0 && ((pcm_stride * esz) & 15) == 0;
  const long long items = B * a.tiles_per_row;
  const int ti = pcm_dtype == WEKWS_PCM_S16 ? 0 : 1;
  const long long cap = (long long)device_sm_count() * h->occ[ti];
  const int grid = (int)(items < cap ? items : cap);
  cudaStream_t st = (cudaStream_t)stream;
  if (ti == 0) resample_kernel<int16_t><<<grid, kRsThreads, h->smem, st>>>(a);
  else resample_kernel<float><<<grid, kRsThreads, h->smem, st>>>(a);
  return check_launch("resample_kernel");
}
