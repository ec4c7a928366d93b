// Streaming front-end state of the reference's online keyword spotter, many streams per call: what
// KeyWordSpotter.accept_wave (wekws/bin/stream_kws_ctc.py:335-398) keeps per stream between chunks --
//   * wave_remained (:347-364): the samples not yet consumed by a whole 10 ms hop, prepended to the next chunk;
//   * feature_remained (:366-390): the last left + right raw feature rows, prepended to the next chunk's rows (the first
//     chunk replicates its first row `left` times instead);
//   * feats_ctx_offset (:391-397): where the next chunk's frame skip starts.
// The host knows every one of these counts (they are integer functions of the chunk lengths) and passes them in; the
// kernels only move the samples and rows, so their output is bit-exact.  One block per stream: a stream's new remainder
// overwrites the old one only after the block has read it.
#include <stdint.h>

#include "common.cuh"

namespace wekws {
namespace {

constexpr int NT = 256;

__global__ void __launch_bounds__(NT) stream_pcm_kernel(const int16_t* __restrict__ chunk, long long chunk_stride,
                                                        const int32_t* __restrict__ chunk_len,
                                                        const int32_t* __restrict__ rem_len,
                                                        const int32_t* __restrict__ consumed, int16_t* remainder,
                                                        long long rem_stride, int16_t* stage, long long stage_stride) {
  const long long b = blockIdx.x;
  const int r = rem_len[b], c = chunk_len[b], cons = consumed[b];
  if (c == 0 && cons == 0) return;                   // no new audio and nothing consumed: the stream does not advance
  const int total = r + c;
  int16_t* rm = remainder + b * rem_stride;
  int16_t* sg = stage + b * stage_stride;
  const int16_t* ch = chunk + b * chunk_stride;
  for (int i = threadIdx.x; i < total; i += NT) sg[i] = i < r ? rm[i] : ch[i - r];    // np.append(wave_remained, wave)
  __syncthreads();
  for (int i = threadIdx.x; i < total - cons; i += NT) rm[i] = sg[cons + i];          // wave[feat_len * frame_shift:]
}

__global__ void __launch_bounds__(NT) stream_context_kernel(const float* __restrict__ feats, long long feat_stride, int D,
                                                            const int32_t* __restrict__ nfeat,
                                                            const int32_t* __restrict__ rem_rows,
                                                            const int32_t* __restrict__ skip_off,
                                                            const int32_t* __restrict__ nout,
                                                            const int32_t* __restrict__ dst_row, int left, int right,
                                                            int skip, float* remainder, float* __restrict__ out) {
  const long long b = blockIdx.x;
  const int F = nfeat[b];
  if (F <= 0) return;
  const int W = left + right + 1, LR = left + right;
  const int r = rem_rows[b];
  const bool first = r == 0;
  const int pre = first ? left : r;                  // padded rows in front of this chunk's features
  const float* f = feats + b * feat_stride * D;
  float* rm = remainder + b * (long long)LR * D;
  const int off = skip_off[b];
  const long long n = (long long)nout[b] * W * D;
  float* o = out + (long long)dst_row[b] * W * D;
  for (long long e = threadIdx.x; e < n; e += NT) {
    const long long j = e / (W * D);
    const int rest = (int)(e - j * W * D);
    const int k = rest / D, d = rest - k * D;
    const long long p = off + j * skip + k;         // row of the padded sequence
    o[e] = p < pre ? (first ? f[d] : rm[p * D + d]) : f[(p - pre) * D + d];
  }
  __syncthreads();
  const int keep = LR < F ? LR : F;                  // feats[-(left + right):] of the un-expanded rows
  for (int e = threadIdx.x; e < keep * D; e += NT) rm[e] = f[(long long)(F - keep) * D + e];
}

}  // namespace
}  // namespace wekws

using namespace wekws;

extern "C" int wekws_stream_pcm(const int16_t* d_chunk, int64_t chunk_stride, int64_t B, const int32_t* d_chunk_len,
                                const int32_t* d_rem_len, const int32_t* d_consumed, int16_t* d_remainder,
                                int64_t rem_stride, int16_t* d_stage, int64_t stage_stride, void* stream) {
  WEKWS_REQUIRE(B >= 0 && B < (1ll << 31) && chunk_stride >= 0 && rem_stride >= 0 && stage_stride >= rem_stride,
                "wekws_stream_pcm: bad sizes");
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE((d_chunk || chunk_stride == 0) && d_chunk_len && d_rem_len && d_consumed && d_remainder && d_stage,
                "wekws_stream_pcm: null argument");
  stream_pcm_kernel<<<(unsigned)B, NT, 0, (cudaStream_t)stream>>>(d_chunk, chunk_stride, d_chunk_len, d_rem_len,
                                                                   d_consumed, d_remainder, rem_stride, d_stage,
                                                                   stage_stride);
  return check_launch("stream_pcm_kernel");
}

extern "C" int wekws_stream_context(const float* d_feats, int64_t feat_stride, int64_t B, int D, const int32_t* d_nfeat,
                                    const int32_t* d_rem_rows, const int32_t* d_skip_off, const int32_t* d_nout,
                                    const int32_t* d_dst_row, int left, int right, int skip, float* d_remainder,
                                    float* d_out, void* stream) {
  WEKWS_REQUIRE(B >= 0 && B < (1ll << 31) && feat_stride >= 0 && D >= 1 && skip >= 1,
                "wekws_stream_context: bad sizes");
  WEKWS_REQUIRE(left == right && left >= 0,
                "wekws_stream_context: left context %d != right context %d is not supported", left, right);
  if (B == 0) return WEKWS_OK;
  WEKWS_REQUIRE(d_feats && d_nfeat && d_rem_rows && d_skip_off && d_nout && d_dst_row &&
                    (d_remainder || left + right == 0),
                "wekws_stream_context: null argument");
  stream_context_kernel<<<(unsigned)B, NT, 0, (cudaStream_t)stream>>>(d_feats, feat_stride, D, d_nfeat, d_rem_rows,
                                                                       d_skip_off, d_nout, d_dst_row, left, right, skip,
                                                                       d_remainder, d_out);
  return check_launch("stream_context_kernel");
}
