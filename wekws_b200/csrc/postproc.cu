// On-device detection statistics for max-pooling keyword models (SURVEY 8f-2): what the reference computes on the
// host from the text score file -- wekws/bin/score.py:128-137 writes every frame's posterior with '{:.6f}',
// wekws/bin/compute_det.py:76-105 then takes, per threshold, (a) max(score_list) < threshold over keyword
// utterances (false rejects) and (b) a left-to-right scan over filler utterances that counts a trigger whenever
// score >= threshold and then skips `window_shift` frames (false alarms).
//
// Bit-exact with that pipeline: a float posterior x in [0, 1] times 1e6 is exact in double (24 x 20 significant
// bits), so rint(x * 1e6) / 1e6 is precisely the double Python parses back from '{:.6f}'.format(x), and the
// thresholds are supplied by the host as the doubles the reference accumulates (threshold += step).
#include <stdint.h>

#include "common.cuh"

namespace wekws {
namespace {

// one thread per (stream b, keyword k, threshold i); a warp covers consecutive thresholds of one (b, k), so the
// posteriors it scans are broadcast loads
__global__ void det_stats_kernel(const float* __restrict__ post, const int32_t* __restrict__ lens, long long B,
                                 long long T, int K, const double* __restrict__ thr, int nthr, int window_shift,
                                 double* __restrict__ max_score, int32_t* __restrict__ triggers) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = B * K * (long long)nthr;
  if (idx >= total) return;
  const int i = (int)(idx % nthr);
  const long long bk = idx / nthr;
  const int k = (int)(bk % K);
  const long long b = bk / K;
  long long n = lens ? (long long)lens[b] : T;
  n = n < 0 ? 0 : (n > T ? T : n);
  const float* p = post + (b * T) * K + k;
  const double th = thr[i];
  int count = 0;
  long long t = 0;
  while (t < n) {                                   // compute_det.py:91-97
    if (text_round6(p[t * K]) >= th) { ++count; t += window_shift; }
    else ++t;
  }
  triggers[idx] = count;
  if (i == 0) {                                     // compute_det.py:83: max(score_list) (as rounded text values)
    float m = -INFINITY;
    for (long long u = 0; u < n; ++u) m = fmaxf(m, p[u * K]);
    max_score[bk] = n > 0 ? text_round6(m) : (double)m;     // the double Python parses back (compared in double)
  }
}

}  // namespace
}  // namespace wekws

using namespace wekws;

extern "C" int wekws_det_stats(const float* d_post, const int32_t* d_lens, int64_t B, int64_t T, int K,
                               const double* d_thresholds, int nthr, int window_shift, double* d_max_score,
                               int32_t* d_triggers, void* stream) {
  WEKWS_REQUIRE(B >= 0 && T >= 0 && K >= 1 && nthr >= 1, "wekws_det_stats: bad sizes");
  WEKWS_REQUIRE(window_shift >= 1, "wekws_det_stats: window_shift must be >= 1 (got %d)", window_shift);
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE((d_post || T == 0) && d_thresholds && d_max_score && d_triggers, "wekws_det_stats: null argument");
  const long long total = (long long)B * K * nthr;
  const int nt = 128;
  det_stats_kernel<<<(unsigned)((total + nt - 1) / nt), nt, 0, (cudaStream_t)stream>>>(
      d_post, d_lens, B, T, K, d_thresholds, nthr, window_shift, d_max_score, d_triggers);
  return check_launch("det_stats_kernel");
}

// ------------------------------------------------------------------------------------------------------------------
// The same rule online: compute_det.py:91-97 over the concatenation of a stream's chunks, resumed each call from a
// two-integer record per (stream, keyword).  After a firing at frame t the scan skips to t + window_shift, which may
// lie in a later chunk, so the record keeps that frame as `next`.
namespace wekws {
namespace {

struct ThresholdState {
  long long seen;   // model frames consumed since reset
  long long next;   // first frame index that may fire
};

// one thread per (stream b, keyword k); the thread owns that pair's record and its event slots, so there are no atomics
__global__ void threshold_spot_kernel(const float* __restrict__ probs, int K, const int32_t* __restrict__ rows,
                                      const int32_t* __restrict__ frames, long long B, const double* __restrict__ thr,
                                      int window_shift, ThresholdState* __restrict__ state, int max_events,
                                      int32_t* __restrict__ counts, wekws_threshold_event* __restrict__ events) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * K) return;
  const long long b = idx / K;
  const int k = (int)(idx - b * K);
  const int n = frames[b];
  int count = 0;
  if (n > 0) {
    ThresholdState s = state[idx];
    const float* p = probs + (long long)rows[b] * K + k;
    const double th = thr[k];
    long long i = s.next > s.seen ? s.next - s.seen : 0;
    while (i < n) {
      const float x = p[i * K];
      if (text_round6(x) >= th) {
        const long long t = s.seen + i;
        if (count < max_events) events[idx * max_events + count] = wekws_threshold_event{t, k, x};
        ++count;
        s.next = t + window_shift;
        i += window_shift;
      } else {
        ++i;
      }
    }
    s.seen += n;
    state[idx] = s;
  }
  counts[idx] = count;
}

}  // namespace
}  // namespace wekws

static_assert(sizeof(wekws_threshold_event) == 16, "wekws_threshold_event layout is part of the C ABI");

extern "C" int64_t wekws_threshold_spot_state_bytes(void) { return (int64_t)sizeof(ThresholdState); }

extern "C" int wekws_threshold_spot(const float* d_probs, int K, const int32_t* d_rows, const int32_t* d_frames,
                                    int64_t B, const double* d_thresholds, int window_shift, void* d_state,
                                    int max_events, int32_t* d_counts, wekws_threshold_event* d_events, void* stream) {
  WEKWS_REQUIRE(B >= 0 && B < (1ll << 31) && K >= 1 && K <= 65535, "wekws_threshold_spot: bad sizes");
  WEKWS_REQUIRE(window_shift >= 1, "wekws_threshold_spot: window_shift must be >= 1 (got %d)", window_shift);
  WEKWS_REQUIRE(max_events >= 0, "wekws_threshold_spot: max_events must be >= 0");
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_probs && d_rows && d_frames && d_thresholds && d_state && d_counts &&
                    (d_events || max_events == 0),
                "wekws_threshold_spot: null argument");
  const long long total = (long long)B * K;
  const int nt = 128;
  threshold_spot_kernel<<<(unsigned)((total + nt - 1) / nt), nt, 0, (cudaStream_t)stream>>>(
      d_probs, K, d_rows, d_frames, B, d_thresholds, window_shift, (ThresholdState*)d_state, max_events, d_counts,
      d_events);
  return check_launch("threshold_spot_kernel");
}

// ------------------------------------------------------------------------------------------------------------------
// Input transforms of the FSMN / CTC recipes (SURVEY 8f-4): context expansion + frame skipping, i.e.
// wekws/dataset/processor.py:267-312 (context_expansion, frame_skip; batched twin wekws/dataset/init_dataset.py:24-68):
//   ctx[t] = concat(feats[max(t - left, 0)], ..., feats[t], ..., feats[t + right])   for t < n - right
//   (the roll() wrap-around on the left is overwritten by the first frame -- "replication pad left margin" -- and the
//   last `right` frames are dropped, so nothing ever wraps), then every skip_rate-th frame is kept.
namespace wekws {
namespace {
__global__ void context_expand_kernel(const float* __restrict__ feats, const int32_t* __restrict__ lens, long long B,
                                      long long T, int D, int left, int right, int skip, float* __restrict__ out,
                                      long long out_frames) {
  const int W = left + right + 1;
  const long long row = blockIdx.x;                 // (b, i)
  const long long b = row / out_frames, i = row - b * out_frames;
  long long n = lens ? (long long)lens[b] : T;
  n = n < 0 ? 0 : (n > T ? T : n);
  const long long kept = n > right ? (n - right + skip - 1) / skip : 0;
  float* o = out + row * (long long)W * D;
  const float* f = feats + b * T * D;
  for (int e = threadIdx.x; e < W * D; e += blockDim.x) {
    float v = 0.f;
    if (i < kept) {
      const int idx = e / D, d = e - idx * D;
      long long t = i * skip + idx - left;
      if (t < 0) t = 0;
      v = f[t * D + d];
    }
    o[e] = v;
  }
}
}  // namespace
}  // namespace wekws

extern "C" int64_t wekws_context_expand_frames(int64_t num_frames, int right, int skip) {
  if (skip < 1 || right < 0 || num_frames <= right) return 0;
  return (num_frames - right + skip - 1) / skip;
}

extern "C" int wekws_context_expand(const float* d_feats, const int32_t* d_lens, int64_t B, int64_t T, int D, int left,
                                    int right, int skip, float* d_out, int64_t out_frames, void* stream) {
  WEKWS_REQUIRE(B >= 0 && T >= 0 && D >= 1 && left >= 0 && right >= 0 && skip >= 1, "wekws_context_expand: bad sizes");
  WEKWS_REQUIRE(out_frames >= wekws_context_expand_frames(T, right, skip), "wekws_context_expand: out_frames %lld too small",
                (long long)out_frames);
  if (B == 0 || out_frames == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_out && (d_feats || T == 0), "wekws_context_expand: null argument");
  WEKWS_REQUIRE(B * out_frames < (1ll << 31), "wekws_context_expand: too many output rows");
  context_expand_kernel<<<(unsigned)(B * out_frames), 128, 0, (cudaStream_t)stream>>>(d_feats, d_lens, B, T, D, left,
                                                                                     right, skip, d_out, out_frames);
  return check_launch("context_expand_kernel");
}
