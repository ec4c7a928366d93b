// Fused Kaldi-compatible log-mel filterbank (+ optional CMVN) for batches of PCM streams.
//
// Replaces torchaudio.compliance.kaldi.fbank as called from the reference
// (wekws/dataset/processor.py:196-202, wekws/bin/stream_kws_ctc.py:354-360) and
// GlobalCMVN.forward (wekws/model/cmvn.py:45-47): snip-edges framing (kaldi.py:44-83),
// per-frame DC removal -> pre-emphasis with replicate padding -> window -> zero pad to 512
// (kaldi.py:183-211), |rfft|^2 (kaldi.py:616-618), sparse triangular mel projection
// (kaldi.py:436-511, 630), log(max(., eps)) (kaldi.py:633).
//
// One warp owns one frame for the FFT.  The 512-point real FFT is a 256-point complex FFT of the
// even/odd packed frame, done as a radix-8 / radix-8 / radix-4 Stockham autosort with the
// first radix-8 entirely in registers (lane p holds z[p + 32 r]), two exchanges through one
// padded per-warp shared buffer of (re, im) pairs (8-byte accesses), and the real-FFT untangle by warp shuffles;
// lane-constant twiddles live in registers.  A CTA (8 warps) stages the 5360 samples its 32
// consecutive frames need once (16-byte loads, converted to float; the next item's vectors are prefetched),
// so each PCM byte is read from HBM ~1.05x and each output byte written once.  The log-mel kernel
// is sized for THREE CTAs per SM (75.9 KB of shared memory, <= 80 registers): 24 warps hide the
// shared-memory and shuffle latencies of the FFT better than the 16 of the mid-round-2 kernel.
// The mel projection runs after all 32 power spectra of the work item are in shared memory, with
// lane = frame and the (warp-uniform) sparse row of one mel bin per warp, read from the constant bank:
// no divergence between lanes whatever the filter widths.
#include <math.h>
#include <string.h>
#include <vector>

#include "common.cuh"
#include "fbank_core.cuh"

namespace wekws {

namespace {

constexpr int FB_WARPS = 8;                 // warps per CTA
constexpr int FB_FPW = 4;                   // frames per warp per work item
constexpr int FB_FRAMES = FB_WARPS * FB_FPW; // frames per CTA work item (one staging load)
constexpr int FB_NT = FB_WARPS * 32;
using fbcore::WIN; using fbcore::SHIFT; using fbcore::NFFT; using fbcore::NBIN; using fbcore::E_SZ;
constexpr int STAGE = (FB_FRAMES - 1) * SHIFT + WIN;  // 5360 samples
constexpr int MAX_MEL = 128;
constexpr int P_ST = NBIN + 1;              // row pitch of the power-spectrum tile (odd: lane = frame reads are conflict-free)
constexpr int O_ST = MAX_MEL + 4;           // row pitch of the output staging tile (aliases the PCM stage; 16-byte rows)
static_assert(FB_FRAMES == 32, "the mel phase maps one frame to one lane");
static_assert(FB_FRAMES * O_ST <= STAGE, "output staging must fit in the PCM stage");
static_assert(STAGE % 8 == 0, "vector staging");
// shared-memory layout (floats): [PCM stage as float / output tile][exchange buffers][tw512][window]
// [log-mel kernel: power tile | MFCC kernel: mel weights]
constexpr int MW_MAX = 2 * NBIN + 64;       // non-zero mel weights supported (80 bins at 16 kHz: 501)
constexpr int SMEM_FLOATS_COMMON = STAGE + FB_WARPS * 2 * E_SZ + 2 * NBIN + WIN;
static_assert((SMEM_FLOATS_COMMON + FB_FRAMES * P_ST) * 4 + 1024 <= 233472 / 3, "the log-mel kernel must fit three times per SM");

struct FbankArgs {
  const void* pcm;
  const int32_t* lens;
  const float* mean;
  const float* istd;
  float* out;
  long long B, num_samples, pcm_stride, max_frames;
  int nmel;
  float preemph, log_floor;
  float log_of_floor;       // logf(log_floor), evaluated on the host: flooring bins get exactly the reference's constant
  int out_vec_ok;           // output rows are 16-byte aligned multiples of 4 floats: tile rows leave with 16-byte stores
  int remove_dc;
  int vec_ok;               // every stream starts 16-byte aligned: stage PCM with 16-byte loads
  // tables (device)
  const float2* tw256;     // W_256^j
  const float2* tw512;     // W_512^k, k < 256
  const float* window;     // 400
  const int* mstart;       // per mel bin: first fft bin, count, offset into mw
  const int* mcnt;
  const int* moff;
  const float* mw;
  int mw_total;
  // MFCC mode (nceps > 0): out = ((log-mel . dct) * lifter - mean) * istd, dct [nmel][nceps]
  const float* dct;
  const float* lifter;
  int nceps, odim;          // odim = row width of `out` (nceps in MFCC mode, else nmel)
};

// The sparse mel filterbank of the log-mel kernel travels in the kernel-parameter constant bank: in the mel phase a
// warp works on ONE mel bin at a time (lane = frame), so the row's start / length / weights are warp-uniform and come
// through the uniform datapath (LDCU) instead of competing with the per-lane spectrum loads for the shared-memory
// pipe -- and the 3.8 KB of tables they used to occupy there is what lets a third CTA fit on the SM.
// Rows are padded with zero weights to a multiple of 4 taps (a row that would run past bin 255 is shifted left
// instead, with leading zeros), so the mel loop is 4 taps per trip with one 16-byte constant load and no remainder;
// a zero weight adds exactly nothing (the spectra are finite and stay inside the frame's own row).
constexpr int MW_PAD_MAX = MW_MAX + 3 * MAX_MEL;
struct MelTable {
  alignas(16) float w[MW_PAD_MAX];          // padded weights, row after row (every row starts 16-byte aligned)
  int16_t start[MAX_MEL], cnt[MAX_MEL], off[MAX_MEL];   // per mel bin: first fft bin, padded taps, offset into w
};

// Natural logarithm for the log-mel epilogue: MUFU lg2 gives log2(x) to ~2^-22 relative, one Newton step on
// 2^-t x = 1 + delta removes that error (log x = ln2 t + log(1 + delta), |delta| < 1e-5 so log(1 + delta) = delta to
// 1e-11): max error 1.3e-6 at |log x| ~ 16 against 1.1e-6 for libm's logf (float64 truth; profiles/r02_fbank_notes.md), in 6
// instructions instead of 32.  x must be a positive normal float (callers floor at log_floor and route anything else
// to logf).
__device__ __forceinline__ float log_newton(float x) {
  float t, e;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-t));
  return fmaf(0.693147180559945309f, t, fmaf(x, e, -1.0f));
}
// log(max(e, floor)) as kaldi.py:633 computes it
__device__ __forceinline__ float log_floored(float e, float floor_v, float log_of_floor) {
  const float x = fmaxf(e, floor_v);
  if (!(x >= 1.17549435e-38f && x <= 1.0e37f)) return logf(x);        // denormal floor, 2^-t would underflow, inf, nan: never in practice
  return x == floor_v ? log_of_floor : log_newton(x);
}

// MFCC = true adds the cepstral epilogue: the log-mel rows of the warp's FB_FPW frames stay in registers
// (lane owns bins lane + 32 k) and are multiplied with the DCT matrix together, so every matrix element is
// loaded once per FB_FPW frames and 12-16 accumulators run in parallel.
// Training front-end (DITHER, wekws_fbank_forward_dither): Gaussian dither noise enters each frame as it is read from
// the PCM stage (fbcore::frame_power_spectrum, dither.cuh).  Its own parameter block comes after the mel table, so the
// parameter layout, and the code, of the undithered instantiations is what it was before the dithered ones existed.
struct DitherArgs {
  float scale;              // the `dither` of kaldi.fbank
  uint32_t key0, key1;      // 64-bit seed (lo, hi)
};

template <typename PCM, bool MFCC, bool DITHER>
__global__ void __launch_bounds__(FB_NT, (MFCC || DITHER) ? 2 : 3)
fbank_kernel(const FbankArgs a, const __grid_constant__ MelTable mt, const DitherArgs dz) {
  extern __shared__ __align__(16) float fb_smem[];
  float* s_stage = fb_smem;                                              // [STAGE]
  float2* s_ex = reinterpret_cast<float2*>(s_stage + STAGE);              // [FB_WARPS][E_SZ] exchange buffers
  float2* s_tw512 = s_ex + FB_WARPS * E_SZ;                              // 0.5 W_512^k
  float2* s_win = s_tw512 + NBIN;
  float* s_pow = reinterpret_cast<float*>(s_win + WIN / 2);              // [FB_FRAMES][P_ST] (log-mel kernel)
  float* s_mw = s_pow;                                                   // [MW_MAX] (MFCC kernel: per-lane mel rows)

  const int tid = threadIdx.x, lane = tid & 31;
  // warp-uniform for the compiler too: the per-frame branches below are then uniform and the shuffles inside them
  // need no WARPSYNC / collective bracket
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  for (int i = tid; i < NBIN; i += FB_NT) s_tw512[i] = make_float2(0.5f * a.tw512[i].x, 0.5f * a.tw512[i].y);
  for (int i = tid; i < WIN / 2; i += FB_NT) s_win[i] = make_float2(a.window[2 * i], a.window[2 * i + 1]);
  if (MFCC)
    for (int i = tid; i < a.mw_total; i += FB_NT) s_mw[i] = a.mw[i];

  fbcore::LaneTwiddles tw;
  tw.load(a.tw256, lane);

  float2* E = s_ex + warp * E_SZ;
  float* Br = reinterpret_cast<float*>(E);      // MFCC kernel: the frame's power spectrum lands in the (free) exchange buffer

  // Work items: (stream b, block of 32 frames fblk).  Per-stream quantities are 32-bit (the host checks the sizes);
  // a CTA steps through its items by adding (gridDim / nfb, gridDim % nfb) -- no division in the loop.
  const int max_frames = (int)a.max_frames, num_samples = (int)a.num_samples;
  const int nfb = (max_frames + FB_FRAMES - 1) / FB_FRAMES;
  const int items = (int)a.B * nfb;
  const int db = (int)gridDim.x / nfb, dfb = (int)gridDim.x % nfb;
  int b = (int)blockIdx.x / nfb, fblk = (int)blockIdx.x % nfb;
  // int16 log-mel kernel: the 16-byte vectors of the NEXT work item are requested right after the FFT phase and sit in
  // registers through the (register-light) mel and store phases, so the staging at the top of the loop converts data
  // that has already arrived instead of waiting a DRAM round trip with the whole CTA at the barrier.
  constexpr int VW = 16 / (int)sizeof(PCM);       // samples per 16-byte load
  constexpr bool PRE = !MFCC && sizeof(PCM) == 2;
  constexpr int NV = (STAGE / VW + FB_NT - 1) / FB_NT;
  uint4 pre[PRE ? NV : 1];
  auto item_len = [&](int bb) {
    const int len = a.lens ? a.lens[bb] : num_samples;
    return len > num_samples ? num_samples : len;
  };
  auto prefetch = [&](int bb, int fb) {
    const int base = fb * FB_FRAMES * SHIFT, len = item_len(bb);
    const PCM* src = reinterpret_cast<const PCM*>(a.pcm) + (long long)bb * a.pcm_stride;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int i = tid + k * FB_NT;
      const int n = base + i * VW;
      const bool full = i < STAGE / VW && n + VW <= len;     // partial / absent vectors take the scalar path at staging
      pre[k] = full ? __ldg(reinterpret_cast<const uint4*>(src + n)) : make_uint4(0u, 0u, 0u, 0u);
    }
  };
  const bool use_pre = PRE && a.vec_ok;
  if (use_pre && (int)blockIdx.x < items) prefetch(b, fblk);
  auto advance = [&]() {
    fblk += dfb; b += db;
    if (fblk >= nfb) { fblk -= nfb; ++b; }
  };
  for (int item = blockIdx.x; item < items; item += gridDim.x, advance()) {
    const int f0 = fblk * FB_FRAMES;
    const int len = item_len(b);
    int mb = len < WIN ? 0 : 1 + (len - WIN) / SHIFT;
    if (mb > max_frames) mb = max_frames;

    __syncthreads();
    {
      const PCM* src = reinterpret_cast<const PCM*>(a.pcm) + (long long)b * a.pcm_stride;
      const int base = f0 * SHIFT;                  // multiple of 160 samples: 16-byte aligned when the stream is
      if (a.vec_ok) {
#pragma unroll
        for (int k = 0; k < NV; ++k) {
          const int i = tid + k * FB_NT;
          if (i >= STAGE / VW) break;
          const int n = base + i * VW;
          float* d = s_stage + i * VW;
          if (n + VW <= len) {
            const uint4 v = PRE ? pre[PRE ? k : 0] : __ldg(reinterpret_cast<const uint4*>(src + n));
            if (sizeof(PCM) == 2) {
              const uint32_t w[4] = {v.x, v.y, v.z, v.w};
              float f[8];
#pragma unroll
              for (int k = 0; k < 4; ++k) {
                f[2 * k] = (float)(int16_t)(w[k] & 0xffffu);
                f[2 * k + 1] = (float)((int32_t)w[k] >> 16);
              }
              reinterpret_cast<float4*>(d)[0] = make_float4(f[0], f[1], f[2], f[3]);
              reinterpret_cast<float4*>(d)[1] = make_float4(f[4], f[5], f[6], f[7]);
            } else {
              reinterpret_cast<float4*>(d)[0] = make_float4(__uint_as_float(v.x), __uint_as_float(v.y),
                                                            __uint_as_float(v.z), __uint_as_float(v.w));
            }
          } else {
#pragma unroll
            for (int k = 0; k < VW; ++k) d[k] = n + k < len ? (float)src[n + k] : 0.f;
          }
        }
      } else {
        for (int i = tid; i < STAGE; i += FB_NT) {
          const int n = base + i;
          s_stage[i] = n < len ? (float)src[n] : 0.f;
        }
      }
    }
    __syncthreads();

    if (!MFCC) {
      // ---- power spectra of the item's 32 frames -> s_pow ----
      for (int fi = 0; fi < FB_FPW; ++fi) {
        const int fl = warp + FB_WARPS * fi;
        if (f0 + fl < mb) {
          fbcore::frame_power_spectrum<DITHER>(s_stage + fl * SHIFT, s_win, s_tw512, tw, E, s_pow + fl * P_ST,
                                               a.preemph, a.remove_dc, lane, dz.scale, dz.key0, dz.key1, b, f0 + fl);
        }
      }
      __syncthreads();                              // spectra complete; the PCM stage is dead and becomes the output tile
      if (use_pre && item + (int)gridDim.x < items) {
        int nb = b + db, nf = fblk + dfb;
        if (nf >= nfb) { nf -= nfb; ++nb; }
        prefetch(nb, nf);
      }
      // ---- mel projection (sparse rows, kaldi.py:630), log floor, CMVN: lane = frame, one mel bin per warp at a time.
      // Rows of absent frames hold stale values; they are never stored.
      float* s_o = s_stage;
      {
        const float* prow = s_pow + lane * P_ST;
        for (int m = warp; m < a.nmel; m += FB_WARPS) {
          const int st = mt.start[m], cnt4 = mt.cnt[m], off = mt.off[m];     // warp-uniform: constant bank
          const float* p = prow + st;
          float e = 0.f;
#pragma unroll 1
          for (int i = 0; i < cnt4; i += 4) {      // rows are 2 trips on average: no unrolling, no remainder code
            const float4 w = *reinterpret_cast<const float4*>(&mt.w[off + i]);
            e = fmaf(w.x, p[i], e);
            e = fmaf(w.y, p[i + 1], e);
            e = fmaf(w.z, p[i + 2], e);
            e = fmaf(w.w, p[i + 3], e);
          }
          float v = log_floored(e, a.log_floor, a.log_of_floor);
          if (a.mean) v -= __ldg(a.mean + m);
          if (a.istd) v *= __ldg(a.istd + m);
          s_o[lane * O_ST + m] = v;
        }
      }
      __syncthreads();
      for (int fi = 0; fi < FB_FPW; ++fi) {
        const int fl = warp + FB_WARPS * fi;
        const int f = f0 + fl;
        if (f >= max_frames) continue;
        float* outp = a.out + ((long long)b * max_frames + f) * a.odim;
        const bool live = f < mb;
        if (a.out_vec_ok) {                         // nmel <= 128: one 16-byte load + store per lane
          if (4 * lane < a.nmel)
            reinterpret_cast<float4*>(outp)[lane] =
                live ? *reinterpret_cast<const float4*>(s_o + fl * O_ST + 4 * lane) : make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
          for (int m = lane; m < a.nmel; m += 32) outp[m] = live ? s_o[fl * O_ST + m] : 0.f;
        }
      }
      continue;                                     // the barrier at the top of the loop protects s_o
    }

    float lm[FB_FPW][4];                          // MFCC: log-mel rows of this warp's frames (0 for absent frames)
    uint32_t fvalid = 0;
    if (MFCC) {
#pragma unroll
      for (int ff = 0; ff < FB_FPW; ++ff)
#pragma unroll
        for (int k = 0; k < 4; ++k) lm[ff][k] = 0.f;
    }
    for (int fi = 0; fi < FB_FPW; ++fi) {
    const int fl = warp + FB_WARPS * fi;          // frame of this warp within the item
    const int f = f0 + fl;
    if (f >= max_frames) continue;            // warp-uniform; no block barrier inside this loop
    float* outp = a.out + ((long long)b * max_frames + f) * a.odim;
    if (f >= mb) {
      for (int m = lane; m < a.odim; m += 32) outp[m] = 0.f;
      continue;
    }

    fbcore::frame_power_spectrum<DITHER>(s_stage + fl * SHIFT, s_win, s_tw512, tw, E, Br, a.preemph, a.remove_dc, lane,
                                         dz.scale, dz.key0, dz.key1, b, f);
    __syncwarp();
    // ---- mel projection (sparse rows), log floor ----
    {
      fvalid |= 1u << fi;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int m = lane + 32 * k;
        if (m < a.nmel) {
          const int st = __ldg(a.mstart + m), cnt = __ldg(a.mcnt + m);
          const float* w = s_mw + __ldg(a.moff + m);
          float e = 0.f;
          for (int i = 0; i < cnt; ++i) e = fmaf(w[i], Br[st + i], e);
          const float v = log_floored(e, a.log_floor, a.log_of_floor);
#pragma unroll
          for (int ff = 0; ff < FB_FPW; ++ff)
            if (fi == ff) lm[ff][k] = v;          // warp-uniform select keeps the row in registers
        }
      }
    }
    __syncwarp();
    }   // frames of this warp
    // ---- MFCC: DCT-II (torchaudio kaldi.py mfcc: feature.matmul(dct_matrix)), lifter, CMVN ----
    if (MFCC && fvalid != 0) {
      float acc[FB_FPW][4];
#pragma unroll
      for (int ff = 0; ff < FB_FPW; ++ff)
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) acc[ff][cc] = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (32 * k < a.nmel) {
          const int mend = min(32, a.nmel - 32 * k);
#pragma unroll 4
          for (int src = 0; src < mend; ++src) {
            const float* drow = a.dct + (size_t)(32 * k + src) * a.nceps + lane;
            float d[4];
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) d[cc] = lane + 32 * cc < a.nceps ? __ldg(drow + 32 * cc) : 0.f;
#pragma unroll
            for (int ff = 0; ff < FB_FPW; ++ff) {
              const float v = __shfl_sync(0xffffffffu, lm[ff][k], src);
#pragma unroll
              for (int cc = 0; cc < 4; ++cc) acc[ff][cc] = fmaf(v, d[cc], acc[ff][cc]);
            }
          }
        }
      }
#pragma unroll
      for (int ff = 0; ff < FB_FPW; ++ff) {
        if (!((fvalid >> ff) & 1u)) continue;
        float* orow = a.out + ((long long)b * max_frames + f0 + warp + FB_WARPS * ff) * a.odim;
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) {
          const int c = lane + 32 * cc;
          if (c < a.nceps) {
            float v = acc[ff][cc];
            if (a.lifter) v *= __ldg(a.lifter + c);
            if (a.mean) v -= __ldg(a.mean + c);
            if (a.istd) v *= __ldg(a.istd + c);
            orow[c] = v;
          }
        }
      }
    }
  }
}

}  // namespace

}  // namespace wekws

// ------------------------------------------------------------------------------- C ABI
using namespace wekws;

struct wekws_fbank {
  wekws_fbank_config cfg;
  int device = 0;
  float2* d_tw256 = nullptr;
  float2* d_tw512 = nullptr;
  float* d_window = nullptr;
  int* d_mstart = nullptr;
  int* d_mcnt = nullptr;
  int* d_moff = nullptr;
  float* d_mw = nullptr;
  int mw_total = 0;
  MelTable mt;              // host copy of the filterbank rows: passed by value to the log-mel kernel
  int nceps = 0;            // > 0: MFCC mode (wekws_fbank_set_mfcc)
  float* d_dct = nullptr;
  float* d_lifter = nullptr;
};

extern "C" int wekws_fbank_create(const wekws_fbank_config* cfg, const float* h_window,
                                  const float* h_mel, wekws_fbank** out) {
  WEKWS_REQUIRE(cfg && h_window && h_mel && out, "wekws_fbank_create: null argument");
  WEKWS_REQUIRE(cfg->frame_length == WIN && cfg->frame_shift == SHIFT && cfg->n_fft == NFFT,
                "fbank: only frame_length=400, frame_shift=160, n_fft=512 are implemented (got %d/%d/%d)",
                cfg->frame_length, cfg->frame_shift, cfg->n_fft);
  WEKWS_REQUIRE(cfg->num_mel_bins >= 1 && cfg->num_mel_bins <= MAX_MEL, "fbank: num_mel_bins %d out of range",
                cfg->num_mel_bins);
  std::vector<float2> tw256(256), tw512(256);
  const double PI = 3.14159265358979323846;
  for (int j = 0; j < 256; ++j) {
    tw256[j] = make_float2((float)cos(2 * PI * j / 256), (float)-sin(2 * PI * j / 256));
    tw512[j] = make_float2((float)cos(2 * PI * j / 512), (float)-sin(2 * PI * j / 512));
  }
  const int nm = cfg->num_mel_bins;
  std::vector<int> mstart(nm), mcnt(nm), moff(nm);
  std::vector<float> mw;
  for (int m = 0; m < nm; ++m) {
    int first = -1, last = -1;
    for (int k = 0; k < NBIN; ++k)
      if (h_mel[m * NBIN + k] != 0.f) { if (first < 0) first = k; last = k; }
    mstart[m] = first < 0 ? 0 : first;
    mcnt[m] = first < 0 ? 0 : last - first + 1;
    moff[m] = (int)mw.size();
    for (int k = 0; k < mcnt[m]; ++k) mw.push_back(h_mel[m * NBIN + mstart[m] + k]);
  }
  WEKWS_REQUIRE(mw.size() <= (size_t)MW_MAX, "fbank: mel filterbank has %zu non-zeros, more than the %d supported",
                mw.size(), MW_MAX);
  if (mw.empty()) mw.push_back(0.f);
  wekws_fbank* fb = new (std::nothrow) wekws_fbank();
  if (!fb) { set_error("out of host memory"); return WEKWS_ERR_NOMEM; }
  fb->cfg = *cfg;
  fb->mw_total = (int)mw.size();
  memset(&fb->mt, 0, sizeof(fb->mt));
  {
    int used = 0;                                   // padded rows (MelTable): zeros in front if the row is shifted left
    for (int m = 0; m < nm; ++m) {
      const int cnt4 = (mcnt[m] + 3) & ~3;
      int st = mstart[m];
      if (st + cnt4 > NBIN) st = NBIN - cnt4;
      if (st < 0 || used + cnt4 > MW_PAD_MAX) {
        delete fb;
        set_error("fbank: mel filterbank does not fit the padded table");
        return WEKWS_ERR_INVALID;
      }
      for (int k = 0; k < mcnt[m]; ++k) fb->mt.w[used + (mstart[m] - st) + k] = mw[moff[m] + k];
      fb->mt.start[m] = (int16_t)st; fb->mt.cnt[m] = (int16_t)cnt4; fb->mt.off[m] = (int16_t)used;
      used += cnt4;
    }
  }
  WEKWS_CUDA_OK(cudaGetDevice(&fb->device));
#define UP(dst, vec)                                                                      \
  WEKWS_CUDA_OK(cudaMalloc((void**)&dst, vec.size() * sizeof(vec[0])));                   \
  WEKWS_CUDA_OK(cudaMemcpy(dst, vec.data(), vec.size() * sizeof(vec[0]), cudaMemcpyHostToDevice));
  UP(fb->d_tw256, tw256) UP(fb->d_tw512, tw512) UP(fb->d_mstart, mstart) UP(fb->d_mcnt, mcnt)
  UP(fb->d_moff, moff) UP(fb->d_mw, mw)
#undef UP
  WEKWS_CUDA_OK(cudaMalloc((void**)&fb->d_window, WIN * sizeof(float)));
  WEKWS_CUDA_OK(cudaMemcpy(fb->d_window, h_window, WIN * sizeof(float), cudaMemcpyHostToDevice));
  *out = fb;
  return WEKWS_OK;
}

extern "C" void wekws_fbank_destroy(wekws_fbank* fb) {
  if (!fb) return;
  cudaFree(fb->d_tw256); cudaFree(fb->d_tw512); cudaFree(fb->d_window);
  cudaFree(fb->d_mstart); cudaFree(fb->d_mcnt); cudaFree(fb->d_moff); cudaFree(fb->d_mw);
  cudaFree(fb->d_dct); cudaFree(fb->d_lifter);
  delete fb;
}

extern "C" int64_t wekws_fbank_num_frames(const wekws_fbank* fb, int64_t num_samples) {
  const int win = fb ? fb->cfg.frame_length : WIN, shift = fb ? fb->cfg.frame_shift : SHIFT;
  return num_samples < win ? 0 : 1 + (num_samples - win) / shift;
}

extern "C" int wekws_fbank_num_mel_bins(const wekws_fbank* fb) { return fb ? fb->cfg.num_mel_bins : 0; }

extern "C" int wekws_fbank_feature_dim(const wekws_fbank* fb) {
  return !fb ? 0 : fb->nceps > 0 ? fb->nceps : fb->cfg.num_mel_bins;
}

extern "C" int wekws_fbank_set_mfcc(wekws_fbank* fb, int num_ceps, const float* h_dct, const float* h_lifter) {
  WEKWS_REQUIRE(fb, "wekws_fbank_set_mfcc: null handle");
  cudaFree(fb->d_dct); cudaFree(fb->d_lifter);
  fb->d_dct = nullptr; fb->d_lifter = nullptr; fb->nceps = 0;
  if (num_ceps == 0) return WEKWS_OK;               // back to log-mel output
  WEKWS_REQUIRE(h_dct, "wekws_fbank_set_mfcc: null dct matrix");
  WEKWS_REQUIRE(num_ceps >= 1 && num_ceps <= fb->cfg.num_mel_bins, "mfcc: num_ceps %d must be in 1..num_mel_bins (%d)",
                num_ceps, fb->cfg.num_mel_bins);   // torchaudio kaldi.py mfcc: assert num_ceps <= num_mel_bins
  const size_t n = (size_t)fb->cfg.num_mel_bins * num_ceps;
  WEKWS_CUDA_OK(cudaMalloc((void**)&fb->d_dct, n * sizeof(float)));
  WEKWS_CUDA_OK(cudaMemcpy(fb->d_dct, h_dct, n * sizeof(float), cudaMemcpyHostToDevice));
  if (h_lifter) {
    WEKWS_CUDA_OK(cudaMalloc((void**)&fb->d_lifter, num_ceps * sizeof(float)));
    WEKWS_CUDA_OK(cudaMemcpy(fb->d_lifter, h_lifter, num_ceps * sizeof(float), cudaMemcpyHostToDevice));
  }
  fb->nceps = num_ceps;
  return WEKWS_OK;
}

// dz == nullptr: the undithered kernels; else the dithered ones with *dz
static int fbank_launch(wekws_fbank* fb, const void* d_pcm, int pcm_dtype, int64_t B, int64_t num_samples,
                        int64_t pcm_stride, const int32_t* d_lens, const float* d_mean, const float* d_istd, float* d_out,
                        int64_t max_frames, void* stream, const DitherArgs* dz) {
  WEKWS_REQUIRE(fb && d_out, "wekws_fbank_forward: null handle or output");
  WEKWS_REQUIRE(B >= 0 && num_samples >= 0 && max_frames >= 0, "wekws_fbank_forward: negative size");
  WEKWS_REQUIRE(pcm_dtype == WEKWS_PCM_S16 || pcm_dtype == WEKWS_PCM_F32, "wekws_fbank_forward: bad pcm_dtype %d", pcm_dtype);
  WEKWS_REQUIRE(max_frames >= wekws_fbank_num_frames(fb, num_samples) || d_lens,
                "wekws_fbank_forward: max_frames %lld < frames of %lld samples", (long long)max_frames,
                (long long)num_samples);
  if (B == 0 || max_frames == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_pcm, "wekws_fbank_forward: null pcm");
  FbankArgs a;
  a.pcm = d_pcm; a.lens = d_lens; a.mean = d_mean; a.istd = d_istd; a.out = d_out;
  a.B = B; a.num_samples = num_samples; a.pcm_stride = pcm_stride; a.max_frames = max_frames;
  a.nmel = fb->cfg.num_mel_bins; a.preemph = fb->cfg.preemphasis; a.log_floor = fb->cfg.log_floor;
  a.log_of_floor = (float)log((double)fb->cfg.log_floor);
  a.out_vec_ok = (reinterpret_cast<uintptr_t>(d_out) & 15) == 0 && fb->nceps == 0 && fb->cfg.num_mel_bins % 4 == 0;
  a.remove_dc = fb->cfg.remove_dc;
  a.tw256 = fb->d_tw256; a.tw512 = fb->d_tw512; a.window = fb->d_window;
  a.mstart = fb->d_mstart; a.mcnt = fb->d_mcnt; a.moff = fb->d_moff; a.mw = fb->d_mw;
  a.mw_total = fb->mw_total;
  a.dct = fb->d_dct; a.lifter = fb->d_lifter; a.nceps = fb->nceps;
  a.odim = fb->nceps > 0 ? fb->nceps : fb->cfg.num_mel_bins;
  const long long items = B * ((max_frames + FB_FRAMES - 1) / FB_FRAMES);
  WEKWS_REQUIRE(num_samples < (1ll << 31) - STAGE && max_frames < (1ll << 31) - FB_FRAMES && items < (1ll << 31) - 65536,
                "wekws_fbank_forward: %lld samples x %lld streams is more than one call handles (split the batch)",
                (long long)num_samples, (long long)B);
  const bool mf = fb->nceps > 0;
  const int esz = pcm_dtype == WEKWS_PCM_S16 ? 2 : 4;
  const size_t smem = (size_t)(SMEM_FLOATS_COMMON + (mf ? MW_MAX : FB_FRAMES * P_ST)) * sizeof(float);
  a.vec_ok = (reinterpret_cast<uintptr_t>(d_pcm) & 15) == 0 && ((pcm_stride * esz) & 15) == 0;
  int dev = 0;
  WEKWS_CUDA_OK(cudaGetDevice(&dev));
  WEKWS_REQUIRE(dev == fb->device, "fbank handle was created on device %d but the current device is %d", fb->device, dev);
  WEKWS_REQUIRE(dev >= 0 && dev < 64, "fbank: device index %d out of range", dev);
  static int occ_dev[64][8] = {};        // the occupancy is per device
  int* occ = occ_dev[dev];
  const int ti = (pcm_dtype == WEKWS_PCM_S16 ? 0 : 1) + (mf ? 2 : 0) + (dz ? 4 : 0);
  static const void* const kernels[8] = {
      (const void*)fbank_kernel<int16_t, false, false>, (const void*)fbank_kernel<float, false, false>,
      (const void*)fbank_kernel<int16_t, true, false>,  (const void*)fbank_kernel<float, true, false>,
      (const void*)fbank_kernel<int16_t, false, true>,  (const void*)fbank_kernel<float, false, true>,
      (const void*)fbank_kernel<int16_t, true, true>,   (const void*)fbank_kernel<float, true, true>};
  const void* kern = kernels[ti];
  if (occ[ti] == 0) {
    if (const int rc = opt_in_smem(kern, smem)) return rc;
    WEKWS_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[ti], kern, FB_NT, smem));
    if (occ[ti] < 1) occ[ti] = 1;
  }
  const long long cap = (long long)device_sm_count() * occ[ti];
  const int grid = (int)(items < cap ? items : cap);
  cudaStream_t st = (cudaStream_t)stream;
  const DitherArgs d = dz ? *dz : DitherArgs{0.f, 0u, 0u};
  switch (ti) {
    case 0: fbank_kernel<int16_t, false, false><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
    case 1: fbank_kernel<float, false, false><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
    case 2: fbank_kernel<int16_t, true, false><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
    case 3: fbank_kernel<float, true, false><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
    case 4: fbank_kernel<int16_t, false, true><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
    case 5: fbank_kernel<float, false, true><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
    case 6: fbank_kernel<int16_t, true, true><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
    default: fbank_kernel<float, true, true><<<grid, FB_NT, smem, st>>>(a, fb->mt, d); break;
  }
  return check_launch(dz ? "fbank_kernel (dither)" : "fbank_kernel");
}

extern "C" int wekws_fbank_forward(wekws_fbank* fb, const void* d_pcm, int pcm_dtype, int64_t B,
                                   int64_t num_samples, int64_t pcm_stride, const int32_t* d_lens,
                                   const float* d_mean, const float* d_istd, float* d_out,
                                   int64_t max_frames, void* stream) {
  return fbank_launch(fb, d_pcm, pcm_dtype, B, num_samples, pcm_stride, d_lens, d_mean, d_istd, d_out, max_frames,
                      stream, nullptr);
}

extern "C" int wekws_fbank_forward_dither(wekws_fbank* fb, const void* d_pcm, int pcm_dtype, int64_t B,
                                          int64_t num_samples, int64_t pcm_stride, const int32_t* d_lens,
                                          const float* d_mean, const float* d_istd, float* d_out, int64_t max_frames,
                                          float dither, uint64_t seed, void* stream) {
  WEKWS_REQUIRE(dither == dither && fabsf(dither) <= 3.0e38f, "wekws_fbank_forward_dither: dither must be finite");
  const DitherArgs dz{dither, (uint32_t)seed, (uint32_t)(seed >> 32)};
  return fbank_launch(fb, d_pcm, pcm_dtype, B, num_samples, pcm_stride, d_lens, d_mean, d_istd, d_out, max_frames,
                      stream, &dz);
}

// Test hook: the exact normals the dithered kernel adds, out[b][f][j] for j < 400 (one thread per Philox call)
namespace wekws {
namespace {
__global__ void dither_noise_kernel(uint32_t k0, uint32_t k1, long long B, int frames, float* out) {
  const long long calls = B * frames * (WIN / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < calls; i += (long long)gridDim.x * blockDim.x) {
    const int q = (int)(i % (WIN / 4));
    const long long bf = i / (WIN / 4);
    const int f = (int)(bf % frames), b = (int)(bf / frames);
    const float2 n0 = dither::normal_pair(k0, k1, b, f, 2 * q), n1 = dither::normal_pair(k0, k1, b, f, 2 * q + 1);
    reinterpret_cast<float4*>(out)[i] = make_float4(n0.x, n0.y, n1.x, n1.y);
  }
}
}  // namespace
}  // namespace wekws

extern "C" int wekws_dither_noise(uint64_t seed, int64_t B, int64_t frames, float* d_out, void* stream) {
  WEKWS_REQUIRE(B >= 0 && frames >= 0 && B < (1ll << 31) && frames < (1ll << 31), "wekws_dither_noise: bad size");
  if (B == 0 || frames == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_out && (reinterpret_cast<uintptr_t>(d_out) & 15) == 0, "wekws_dither_noise: output must be 16-byte aligned");
  const long long calls = B * frames * (WIN / 4);
  const int grid = (int)((calls + 255) / 256 < 65536 ? (calls + 255) / 256 : 65536);
  dither_noise_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((uint32_t)seed, (uint32_t)(seed >> 32), B, (int)frames,
                                                             d_out);
  return check_launch("dither_noise_kernel");
}
