// Kernel argument block of the CTC prefix beam search (ctc_decode.cu).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/wekws_b200.h"

namespace wekws {

struct CtcArgs {
  const float* probs;        // (B, T, V) softmax posteriors
  const int32_t* lens;       // (B) valid frames or nullptr
  long long B, T;
  int V;
  const int32_t* allowed;    // keyword token set (n_allowed ids) or nullptr / 0 = every token
  int n_allowed;
  int score_beam, path_beam;
  long long frame_offset;    // absolute frame number of row 0 (streaming: total_frames)
  int frame_stride;          // frames per row (streaming: downsampling)
  uint8_t* state;            // B x ctc_state_bytes() carried hypotheses, or nullptr
  int reset_state;
  int32_t* nhyp;             // (B)
  int32_t* overflow;         // (B)
  int32_t* hyp_len;          // (B, path_beam)      -1 = unused slot
  int32_t* hyp_tokens;       // (B, path_beam, WEKWS_CTC_MAX_PREFIX)
  double* hyp_score;         // (B, path_beam)      pb + pnb
  int32_t* node_frame;       // (B, path_beam, WEKWS_CTC_MAX_PREFIX)
  float* node_prob;          // (B, path_beam, WEKWS_CTC_MAX_PREFIX)
};

// Per-stream detection record of the streaming spotter (wekws_ctc_spot_state_bytes).  All zero = a stream that has
// not decoded a frame since reset_all(); the kernel initialises it on the stream's first frame.
struct SpotDet {
  double hit_score;          // KeyWordSpotter.hit_score
  long long total_frames;    // KeyWordSpotter.total_frames
  int32_t last_active_pos;   // KeyWordSpotter.last_active_pos
  int32_t overflow;          // sticky: some prefix outgrew WEKWS_CTC_MAX_PREFIX
  int32_t live;
  int32_t pad;
};

struct SpotArgs {
  const float* probs;        // softmax posteriors; stream b's frames are rows rows[b] .. rows[b] + frames[b] - 1
  const int32_t* rows;       // (B)
  const int32_t* frames;     // (B) frames this call, 0 = stream not touched
  long long B;
  int V;
  const int32_t* allowed;    // keyword token set ({0} + every keyword token)
  int n_allowed;
  const int32_t* kw_tokens;  // keyword k = kw_tokens[kw_off[k] .. kw_off[k + 1])
  const int32_t* kw_off;
  int nkw;
  int score_beam, path_beam;
  int frame_stride;          // downsampling: row t is frame total_frames + t * frame_stride
  double threshold;
  int min_frames, max_frames, interval_frames;
  uint8_t* state;            // B x ctc_state_bytes() hypotheses (the layout ctc_prefix_beam_kernel carries)
  uint8_t* det;              // B x sizeof(SpotDet)
  wekws_ctc_spot_result* result;   // (B)
};

struct StreamScoreArgs {
  const float* probs;        // (B, T, V) softmax posteriors
  const int32_t* lens;       // (B) valid frames
  long long B, T;
  int V;
  const int32_t* allowed;    // keyword token set ({0} + every keyword token)
  int n_allowed;
  const int32_t* kw_tokens;  // keyword k = kw_tokens[kw_off[k] .. kw_off[k + 1])
  const int32_t* kw_off;
  int nkw;
  int score_beam, path_beam;
  int frame_stride;          // frame_skip: row t is frame t * frame_stride
  double threshold;
  int min_frames, max_frames;
  int max_detections;        // records kept per utterance; the count goes on past it
  int32_t* count;            // (B) activations
  wekws_ctc_stream_detection* det;   // (B, max_detections)
  int32_t* overflow;         // (B)
};

size_t ctc_state_bytes();
size_t ctc_spot_state_bytes();
int ctc_stream_score_launch(const StreamScoreArgs& a, cudaStream_t st);
int ctc_spot_launch(const SpotArgs& a, cudaStream_t st);
int ctc_launch(const CtcArgs& a, cudaStream_t st);
int ctc_hit_launch(const int32_t* nhyp, const int32_t* hyp_len, const int32_t* hyp_tokens, const int32_t* node_frame,
                   const float* node_prob, long long B, int path_beam, const int32_t* kw_tokens, const int32_t* kw_off,
                   int nkw, int32_t* hit, double* hit_score, int32_t* start, int32_t* end, cudaStream_t st);

}  // namespace wekws
