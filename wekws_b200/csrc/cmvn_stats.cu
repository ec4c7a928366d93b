// Global CMVN statistics (tools/compute_cmvn_stats.py: per-dimension sum and sum of squares of every feature frame,
// and the frame count) over a (B, max_frames, D) feature batch as wekws_fbank_forward writes it.
//   * cmvn_utt_sums_kernel: one CTA per utterance forms sum x and sum x^2 of each dimension over its first
//     frames[b] rows in double (the square of a float32 is exact in double), in an order fixed by D alone: thread
//     (d, g) sums frames g, g + G, ... (G = 512 / D groups), then the G partial sums are added in g order.
//   * cmvn_fold_kernel adds the per-utterance sums into the persistent accumulator one utterance after the other, so
//     the result depends only on the order of the utterances, never on how they were split into calls.
#include <stdint.h>

#include "common.cuh"

namespace wekws {
namespace {

constexpr int kStatThreads = 512;       // 6 frame groups at D = 80, two CTAs per SM: short dependent add chains
constexpr int kFoldThreads = 128;

// thread (d, g) sums frames g, g + G, ... of dimension d; the G partial sums are then added in g order
__global__ void __launch_bounds__(kStatThreads, 2) cmvn_utt_sums_kernel(const float* __restrict__ feats,
                                                                     long long max_frames, int D,
                                                                     const int32_t* __restrict__ frames,
                                                                     double* __restrict__ sums) {
  __shared__ double red[2 * kStatThreads];
  const long long b = blockIdx.x;
  long long nf = frames[b];
  nf = nf < 0 ? 0 : (nf > max_frames ? max_frames : nf);
  const float* xb = feats + b * max_frames * D;
  const int Dp = D < kStatThreads ? D : kStatThreads, G = kStatThreads / Dp;
  const int dl = threadIdx.x % Dp, g = threadIdx.x / Dp;
  for (int d0 = 0; d0 < D; d0 += Dp) {
    const int d = d0 + dl;
    double s = 0.0, q = 0.0;
    if (g < G && d < D)
      for (long long t = g; t < nf; t += G) {
        const double v = xb[t * D + d];
        s += v;
        q = fma(v, v, q);
      }
    __syncthreads();
    if (g < G) { red[g * Dp + dl] = s; red[(G + g) * Dp + dl] = q; }
    __syncthreads();
    if (g == 0 && d < D) {
      double ts = red[dl], tq = red[G * Dp + dl];
      for (int k = 1; k < G; ++k) { ts += red[k * Dp + dl]; tq += red[(G + k) * Dp + dl]; }
      sums[b * 2 * D + d] = ts;
      sums[b * 2 * D + D + d] = tq;
    }
  }
}

__global__ void __launch_bounds__(kFoldThreads) cmvn_fold_kernel(const double* __restrict__ sums, long long B, int D,
                                                                 long long max_frames,
                                                                 const int32_t* __restrict__ frames,
                                                                 double* __restrict__ acc,
                                                                 long long* __restrict__ frame_num) {
  const int d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d < D) {
    double s = acc[d], q = acc[D + d];
#pragma unroll 8
    for (long long b = 0; b < B; ++b) {       // unrolled so the loads run ahead of the dependent adds
      s += sums[b * 2 * D + d];
      q += sums[b * 2 * D + D + d];
    }
    acc[d] = s;
    acc[D + d] = q;
  }
  if (d == 0) {
    long long n = *frame_num;
    for (long long b = 0; b < B; ++b) {
      const long long f = frames[b];
      n += f < 0 ? 0 : (f > max_frames ? max_frames : f);
    }
    *frame_num = n;
  }
}

}  // namespace
}  // namespace wekws

using namespace wekws;

extern "C" int64_t wekws_cmvn_stats_workspace_bytes(int64_t B, int D) {
  return B <= 0 || D <= 0 ? 0 : B * 2 * (int64_t)D * (int64_t)sizeof(double);
}

extern "C" int wekws_cmvn_stats_accumulate(const float* d_feats, int64_t B, int64_t max_frames, int D,
                                           const int32_t* d_frames, double* d_acc, int64_t* d_frame_num,
                                           void* d_workspace, void* stream) {
  WEKWS_REQUIRE(B >= 0 && max_frames >= 0 && D >= 1, "wekws_cmvn_stats_accumulate: bad size (B %lld, frames %lld, D %d)",
                (long long)B, (long long)max_frames, D);
  WEKWS_REQUIRE(d_acc && d_frame_num, "wekws_cmvn_stats_accumulate: null accumulator");
  WEKWS_REQUIRE(B < (1ll << 31), "wekws_cmvn_stats_accumulate: %lld utterances is more than one call handles",
                (long long)B);
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_frames && d_workspace && (d_feats || max_frames == 0),
                "wekws_cmvn_stats_accumulate: null features, frame counts or workspace");
  cudaStream_t st = (cudaStream_t)stream;
  double* sums = static_cast<double*>(d_workspace);
  cmvn_utt_sums_kernel<<<(unsigned)B, kStatThreads, 0, st>>>(d_feats, max_frames, D, d_frames, sums);
  int rc = check_launch("cmvn_utt_sums_kernel");
  if (rc != WEKWS_OK) return rc;
  cmvn_fold_kernel<<<(D + kFoldThreads - 1) / kFoldThreads, kFoldThreads, 0, st>>>(sums, B, D, max_frames, d_frames,
                                                                                   d_acc, (long long*)d_frame_num);
  return check_launch("cmvn_fold_kernel");
}
