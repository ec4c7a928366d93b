/*
 * wekws_b200 -- C ABI of the H100-native WeKws streaming keyword-spotting forward path.
 *
 * Plain C, no torch / ATen / C++ types cross this boundary.  Every pointer named
 * d_* is a device pointer on the CURRENT CUDA device; h_* is a host pointer.
 * `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 * Every function returns 0 on success and a negative wekws_status on failure;
 * wekws_last_error() then holds a thread-local human-readable message.  Nothing
 * throws, nothing allocates device memory inside a *_forward call except a
 * per-handle scratch buffer that grows monotonically on first use.
 *
 * What each entry point replaces in the reference (wenet-e2e/wekws @ 1a8ee65):
 *
 *   wekws_fbank_*          torchaudio.compliance.kaldi.fbank as called by
 *                          wekws/dataset/processor.py:173-203 (compute_fbank) and
 *                          wekws/bin/stream_kws_ctc.py:335-364 (accept_wave), fused with
 *                          GlobalCMVN.forward wekws/model/cmvn.py:37-48; native twin:
 *                          wenet::Fbank::Compute runtime/core/frontend/fbank.h:138-198
 *                          behind FeaturePipeline::AcceptWaveform
 *                          runtime/core/frontend/feature_pipeline.cc:30-47.
 *   wekws_model_create /   init_model(configs) wekws/model/kws_model.py:97-214 followed by
 *   _set_tensor/_finalize  load_checkpoint -> load_state_dict wekws/utils/checkpoint.py:23-36;
 *                          tensor names ARE the reference state_dict keys (SURVEY.md 8b).
 *   wekws_model_forward    KWSModel.forward(x, in_cache) wekws/model/kws_model.py:65-76
 *                          (and forward_softmax :78-90 via WEKWS_ACT_SIGMOID/IDENTITY +
 *                          WEKWS_FWD_SOFTMAX); native twin: KeywordSpotting::Forward
 *                          runtime/core/kws/keyword_spotting.cc:56-95 whose ONNX graph has
 *                          inputs (input, cache) and outputs (output, r_cache).
 *   wekws_pipeline_forward the composition the callers perform: Fbank -> model, i.e.
 *                          stream_kws_ctc.py:482-487 / score.py:117-127, raw PCM in,
 *                          posteriors out.
 *   wekws_stream_pcm /     the per-stream state of KeyWordSpotter.accept_wave
 *   wekws_stream_context / wekws/bin/stream_kws_ctc.py:335-398 (PCM remainder, context remainder,
 *   wekws_ctc_spot         frame-skip offset) and the frame loop of KeyWordSpotter.forward :400-514
 *                          (beam-search step, execute_detection, resets), for many streams per call.
 *   wekws_ctc_stream_score the per-utterance frame loop of wekws/bin/stream_score_ctc.py:221-377 (streaming
 *                          decode with its own detection rule over whole utterances of a test set).
 */
#ifndef WEKWS_B200_H_
#define WEKWS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WEKWS_B200_ABI_VERSION 9   /* 2: + wekws_fbank_set_mfcc, wekws_fbank_feature_dim, wekws_det_stats; 3: det max_score is double; 4: precision mode 2, wekws_model_uses_tensor_cores_bt; 5: wekws_model_set_head; 6: + wekws_stream_pcm, wekws_stream_context, wekws_ctc_spot, wekws_ctc_spot_state_bytes; 7: + wekws_ctc_stream_score, wekws_ctc_stream_detection; 8: + wekws_criterion_*; 9: + wekws_resample_*, wekws_cmvn_stats_* */

#if defined(__GNUC__)
#define WEKWS_API __attribute__((visibility("default")))
#else
#define WEKWS_API
#endif

typedef enum {
  WEKWS_OK = 0,
  WEKWS_ERR_INVALID = -1,     /* bad argument / unsupported configuration              */
  WEKWS_ERR_CUDA = -2,        /* a CUDA runtime call failed (message has the string)  */
  WEKWS_ERR_STATE = -3,       /* call order: forward before finalize, missing tensor  */
  WEKWS_ERR_NOMEM = -4
} wekws_status;

typedef enum {
  WEKWS_BACKBONE_MDTC = 0,    /* wekws/model/mdtc.py  MDTC                             */
  WEKWS_BACKBONE_TCN = 1,     /* wekws/model/tcn.py   TCN(block_class=CnnBlock)        */
  WEKWS_BACKBONE_DSTCN = 2,   /* wekws/model/tcn.py   TCN(block_class=DsCnnBlock)      */
  WEKWS_BACKBONE_GRU = 3,     /* torch.nn.GRU, kws_model.py:128-133                    */
  WEKWS_BACKBONE_FSMN = 4     /* wekws/model/fsmn.py FSMN (preprocessing none, classifier identity,
                                 kws_model.py:158-170,121-122,191): tensors backbone.in_linear{1,2}.linear.*,
                                 backbone.fsmn.{l}.{0.linear.weight,1.conv_left.weight,1.conv_right.weight,
                                 2.linear.*}, backbone.out_linear{1,2}.linear.*                    */
} wekws_backbone;

typedef enum { WEKWS_ACT_IDENTITY = 0, WEKWS_ACT_SIGMOID = 1 } wekws_activation;
/* Classifier head (kws_model.py:175-195).  LINEAR: classifier.linear.* on every frame, output (B, T, odim).
 * GLOBAL / LAST: the utterance-level heads of the speech-command recipes (classifier.py:19-40): the MLP
 * Linear(hidden, 64) -> ReLU -> Linear(64, odim) (tensors classifier.classifier.0.{weight,bias} and
 * classifier.classifier.3.{weight,bias}) on the mean of all T frames of the call (GLOBAL) or on frame T-1 (LAST);
 * output (B, odim).  MDTC, TCN and DS-TCN backbones only.                                                     */
typedef enum { WEKWS_HEAD_LINEAR = 0, WEKWS_HEAD_GLOBAL = 1, WEKWS_HEAD_LAST = 2 } wekws_head;
typedef enum { WEKWS_PCM_S16 = 0, WEKWS_PCM_F32 = 1 } wekws_pcm_dtype;
typedef enum { WEKWS_WINDOW_POVEY = 0, WEKWS_WINDOW_HAMMING = 1 } wekws_window;

/* forward flags */
#define WEKWS_FWD_SOFTMAX 1u  /* apply softmax over odim after the activation (forward_softmax); with a GLOBAL /
                                 LAST head it normalises each of the B output rows                               */

WEKWS_API const char* wekws_last_error(void);
WEKWS_API int wekws_abi_version(void);
/* Number of kernels this library has launched since load (all handles, all threads). */
WEKWS_API uint64_t wekws_launch_count(void);

/* ----------------------------------------------------------------------------- Fbank */
typedef struct wekws_fbank wekws_fbank;

typedef struct {
  int32_t sample_rate;     /* 16000                                                   */
  int32_t frame_length;    /* samples per frame, 400  (frame_length=25 ms)            */
  int32_t frame_shift;     /* samples per hop,   160  (frame_shift=10 ms)             */
  int32_t n_fft;           /* 512 (round_to_power_of_two); only 512 is implemented    */
  int32_t num_mel_bins;    /* <= 128                                                  */
  float   preemphasis;     /* 0.97                                                    */
  int32_t remove_dc;       /* 1                                                       */
  float   log_floor;       /* FLT_EPSILON (kaldi.py:21)                               */
} wekws_fbank_config;

/* h_window: frame_length floats (Povey / Hamming, computed by the host exactly as
 * kaldi.py:88-110 does).  h_mel: num_mel_bins x (n_fft/2) row-major mel weights
 * (kaldi.py:436-511; the Nyquist column is implicitly zero, kaldi.py:627).        */
WEKWS_API int wekws_fbank_create(const wekws_fbank_config* cfg, const float* h_window,
                       const float* h_mel, wekws_fbank** out);
WEKWS_API void wekws_fbank_destroy(wekws_fbank* fb);
/* Frames produced for num_samples samples (snip_edges=True): 0 if < frame_length.   */
WEKWS_API int64_t wekws_fbank_num_frames(const wekws_fbank* fb, int64_t num_samples);
WEKWS_API int wekws_fbank_num_mel_bins(const wekws_fbank* fb);

/* MFCC mode (SURVEY 8f-1): the front-end of the shipped mdtc / mdtc_small configs
 * (examples/hi_xiaowen/s0/conf/mdtc.yaml:8-14 `feature_type: mfcc`), i.e.
 * torchaudio.compliance.kaldi.mfcc as called by wekws/dataset/processor.py:157-166 (compute_mfcc):
 * the log-mel row times a DCT-II matrix h_dct[num_mel_bins][num_ceps] (ortho, first column sqrt(1/num_mel_bins)),
 * times h_lifter[num_ceps] (NULL = no liftering), then the optional CMVN of wekws_fbank_forward over the
 * num_ceps outputs.  After this call wekws_fbank_forward writes (B, max_frames, num_ceps).  num_ceps = 0
 * switches back to log-mel output.  wekws_fbank_feature_dim = row width of the output in the current mode. */
WEKWS_API int wekws_fbank_set_mfcc(wekws_fbank* fb, int num_ceps, const float* h_dct, const float* h_lifter);
WEKWS_API int wekws_fbank_feature_dim(const wekws_fbank* fb);

/* d_pcm: B waveforms, row b at d_pcm + b*pcm_stride elements, int16-scale values.
 * d_lens: optional per-waveform sample counts (NULL = all num_samples).
 * d_mean/d_istd: optional CMVN (NULL, NULL = none; istd NULL = mean only).
 * d_out: (B, max_frames, num_mel_bins) fp32; rows past a waveform's frame count are
 * zero-filled.  max_frames must be >= wekws_fbank_num_frames(num_samples).          */
WEKWS_API int wekws_fbank_forward(wekws_fbank* fb, const void* d_pcm, int pcm_dtype, int64_t B,
                        int64_t num_samples, int64_t pcm_stride, const int32_t* d_lens,
                        const float* d_mean, const float* d_istd, float* d_out,
                        int64_t max_frames, void* stream);

/* ----------------------------------------------------------------------------- model */
typedef struct wekws_model wekws_model;

typedef struct {
  int32_t backbone;        /* wekws_backbone                                           */
  int32_t idim;            /* input_dim  (<= 128)                                      */
  int32_t hdim;            /* hidden_dim: 32/64/128/256 for conv backbones, 128 GRU    */
  int32_t odim;            /* output_dim                                               */
  int32_t num_layers;      /* TCN/DSTCN blocks or GRU layers; MDTC: ignored            */
  int32_t num_stack;       /* MDTC only                                                */
  int32_t stack_size;      /* MDTC only                                                */
  int32_t kernel_size;     /* conv taps (mdtc 5, tcn 8)                                */
  int32_t activation;      /* wekws_activation                                         */
  int32_t norm_var;        /* cmvn.norm_var; used when global_cmvn.* tensors are set   */
  /* FSMN only (fsmn_ctc.yaml:40-52); num_layers = FSMN layers; the memory blocks always use strides 1,1 as the
   * reference builds them (fsmn.py:384-391); cache (B, proj_dim, left_order - 1 + right_order, num_layers)  */
  int32_t fsmn_input_affine_dim, fsmn_linear_dim, fsmn_proj_dim;
  int32_t fsmn_left_order, fsmn_right_order, fsmn_output_affine_dim;
} wekws_model_config;

WEKWS_API int wekws_model_create(const wekws_model_config* cfg, wekws_model** out);
WEKWS_API void wekws_model_destroy(wekws_model* m);
/* Total cache columns == backbone.padding (mdtc 244, tcn/ds_tcn 105; FSMN lorder-1+rorder); 0 for GRU. */
WEKWS_API int wekws_model_padding(const wekws_model* m);
/* name: reference state_dict key, e.g. "backbone.blocks.0.res_blocks.1.bn1.running_var".
 * Data is copied.  num_batches_tracked entries may be skipped.                      */
WEKWS_API int wekws_model_set_tensor(wekws_model* m, const char* name, const float* h_data, int64_t numel);
/* head: wekws_head.  Called between create and pack / finalize (default WEKWS_HEAD_LINEAR).  GLOBAL / LAST need an
 * MDTC, TCN or DS-TCN backbone (else WEKWS_ERR_INVALID); the MLP width is 64.  The streaming cache is unchanged. */
WEKWS_API int wekws_model_set_head(wekws_model* m, int head);
/* Host half of finalize: folds every eval-mode BatchNorm into its producer and packs the
 * weight stream.  No CUDA call -- usable (and tested) on a machine without a GPU.        */
WEKWS_API int wekws_model_pack(wekws_model* m);
/* wekws_model_pack + upload to the current device.                                       */
WEKWS_API int wekws_model_finalize(wekws_model* m);
/* Arithmetic of the dense GEMMs: 0 = auto (default): wgmma tensor cores with a 3-pass bf16
 * operand split (~2^-17 relative, posteriors within 1e-5 of fp32) where a fused tensor-core
 * kernel exists (mdtc / dense tcn with hidden 64, ds_tcn with hidden 256 and k = 8; chunk >= 8 frames),
 * FP32 FMA elsewhere; the GRU (hidden 128, 1-2 layers) has a weight-streaming tensor-core kernel that auto picks by batch
 * and chunk (>= 640 streams at T = 1, >= 400 at T = 2..7, >= 256 at T >= 8) and the FP32 kernel otherwise; 1 = FP32 FMA only;
 * 2 = the tensor-core kernel wherever one exists, whatever the batch (tests, benchmarks). */
WEKWS_API int wekws_model_set_precision(wekws_model* m, int mode);
/* 1 if a forward with T frames per call runs a tensor-core kernel (after finalize), else 0.  The plain form answers for
 * a large batch; the GRU's choice also depends on the batch B.                               */
WEKWS_API int wekws_model_uses_tensor_cores(const wekws_model* m, int64_t T);
WEKWS_API int wekws_model_uses_tensor_cores_bt(const wekws_model* m, int64_t B, int64_t T);
/* Debug/test accessors of the packed host-side program (valid after finalize).      */
WEKWS_API int64_t wekws_model_packed_floats(const wekws_model* m, int which /*0 stream, 1 vectors, 2 tensor-core weight images (bytes / 4)*/);
WEKWS_API int wekws_model_packed_copy(const wekws_model* m, int which, float* h_dst, int64_t capacity);

/* d_feats (B,T,idim); d_in_cache NULL (start of stream == zeros) or
 * conv: (B,hdim,padding)  GRU: (num_layers,B,hdim)  FSMN: (B,proj_dim,padding,num_layers); d_out (B,T,odim), or
 * (B,odim) with a GLOBAL / LAST head (pooled over the T frames of this call);
 * d_out_cache same shape as the cache; it may be the SAME buffer as d_in_cache (in-place
 * streaming update: every slice is read before it is overwritten) or a disjoint one, not a
 * partially overlapping one.                                                       */
WEKWS_API int wekws_model_forward(wekws_model* m, const float* d_feats, const float* d_in_cache,
                        float* d_out, float* d_out_cache, int64_t B, int64_t T,
                        uint32_t flags, void* stream);

/* Detection statistics of max-pooling keyword models on the device (SURVEY 8f-2), bit-exact with the host
 * pipeline wekws/bin/score.py:128-137 ('{:.6f}' score file) -> wekws/bin/compute_det.py:76-105:
 *   d_max_score[b,k]   = max over the first lens[b] frames of the text-rounded posterior as the DOUBLE Python parses
 *                        back from the score file (false-reject test `max < threshold` is done in double),
 *   d_triggers[b,k,i]  = triggers of the left-to-right scan "score >= thresholds[i] -> count, skip window_shift
 *                        frames" (false alarms).
 * d_post (B,T,K) posteriors; d_lens NULL = all T frames; d_thresholds nthr doubles (the host accumulates
 * threshold += step exactly as the reference does).                                                   */
WEKWS_API int wekws_det_stats(const float* d_post, const int32_t* d_lens, int64_t B, int64_t T, int K,
                    const double* d_thresholds, int nthr, int window_shift, double* d_max_score,
                    int32_t* d_triggers, void* stream);

/* CTC prefix beam search + keyword look-up on the device (SURVEY 8f-2, CTC models), bit-exact with the reference's pure
 * Python: wekws/model/loss.py:206-312 ctc_prefix_beam_search as called by wekws/bin/score_ctc.py:198-200 (whole
 * utterance) and its per-frame streaming twin wekws/bin/stream_kws_ctc.py:124-215,400-409 (hypotheses carried in
 * d_state between calls; frame numbers = frame_offset + row * frame_stride), then the look-up of
 * score_ctc.py:201-220 / stream_kws_ctc.py:411-434.
 *   d_probs (B,T,V) softmax posteriors; d_lens NULL = T frames; d_keyword_tokens: the keywords' token-id set
 *   (n = 0: no filter); d_state: B x wekws_ctc_state_bytes() bytes or NULL (reset_state != 0: start from the empty
 *   hypothesis and write the final state).
 * Outputs per utterance, hypotheses in beam order: d_nhyp (B); d_hyp_len (B,path_beam) (-1 = unused);
 *   d_hyp_tokens / d_node_frame / d_node_prob (B,path_beam,WEKWS_CTC_MAX_PREFIX); d_hyp_score (B,path_beam) = pb + pnb
 *   (double, as Python computes it); d_overflow (B) != 0 if a prefix outgrew WEKWS_CTC_MAX_PREFIX tokens.          */
#define WEKWS_CTC_MAX_PREFIX 64
#define WEKWS_CTC_MAX_PATH_BEAM 20
#define WEKWS_CTC_MAX_SCORE_BEAM 3
WEKWS_API int64_t wekws_ctc_state_bytes(void);
WEKWS_API int wekws_ctc_prefix_beam_search(const float* d_probs, const int32_t* d_lens, int64_t B, int64_t T, int V,
                                 const int32_t* d_keyword_tokens, int n_keyword_tokens, int score_beam_size,
                                 int path_beam_size, int64_t frame_offset, int frame_stride, void* d_state,
                                 int reset_state, int32_t* d_nhyp, int32_t* d_hyp_len, int32_t* d_hyp_tokens,
                                 double* d_hyp_score, int32_t* d_node_frame, float* d_node_prob, int32_t* d_overflow,
                                 void* stream);
/* d_kw_tokens: the keywords' token sequences back to back, keyword k = [d_kw_offsets[k], d_kw_offsets[k+1]).
 * d_hit (B) = index of the detected keyword or -1; d_hit_score = sqrt(product of its token probabilities);
 * d_start / d_end = frames of its first / last token.                                                        */
WEKWS_API int wekws_ctc_keyword_hit(const int32_t* d_nhyp, const int32_t* d_hyp_len, const int32_t* d_hyp_tokens,
                          const int32_t* d_node_frame, const float* d_node_prob, int64_t B, int path_beam_size,
                          const int32_t* d_kw_tokens, const int32_t* d_kw_offsets, int num_keywords, int32_t* d_hit,
                          double* d_hit_score, int32_t* d_start, int32_t* d_end, void* stream);

/* Streaming keyword spotter (wekws/bin/stream_kws_ctc.py:400-514, KeyWordSpotter.forward after the model call): for
 * every stream with d_frames[b] > 0, frames t = 0 .. d_frames[b]-1 at rows d_rows[b] + t of d_probs (row width V), one
 * step of the streaming prefix beam search (decode_keywords :400-409, hypotheses truncated to path_beam_size) and then
 * execute_detection (:411-480: first hypothesis in beam order containing a keyword in keyword order, hit_score *=
 * token probabilities then sqrt, carried across frames; activation needs hit_score >= threshold,
 * min_frames <= end - start <= max_frames and last_active_pos == -1 or end - last_active_pos >= interval_frames).  On
 * activation the result is recorded, reset() runs (hypotheses, hit_score) and the rest of the chunk is skipped
 * (:495-501).  After the chunk total_frames += d_frames[b] * frame_stride and the max_frames reset of :509-512 runs.
 * Frame numbers are total_frames + t * frame_stride.  Streams with d_frames[b] <= 0 are not touched.
 *   d_keyword_tokens: {0} + every keyword token (set_keywords :304-333); d_kw_tokens / d_kw_offsets: the keywords'
 *   token sequences back to back, keyword k = [d_kw_offsets[k], d_kw_offsets[k+1]), each <= WEKWS_CTC_MAX_PREFIX.
 *   d_state: B x wekws_ctc_state_bytes() hypotheses in the layout of wekws_ctc_prefix_beam_search's d_state (so that
 *   call with T = 0 and reset_state = 0 reads them out); d_det: B x wekws_ctc_spot_state_bytes() detection record
 *   (hit_score, total_frames, last_active_pos, overflow).  A zero d_det row is a stream after reset_all() (:521-529):
 *   its hypotheses are (re)initialised on its first frame, whatever d_state holds.
 *   d_result[b] (written only for streams with frames) is self.result after the last frame processed: state 1 with
 *   keyword index, start / end frames and score on activation, else state 0; overflow != 0 if any prefix of the
 *   stream ever outgrew WEKWS_CTC_MAX_PREFIX tokens.                                                              */
typedef struct {
  double score;            /* hit_score at activation                                   */
  int32_t state;           /* 1 = activated in this chunk                               */
  int32_t keyword;         /* index into the keyword list, -1 if not activated          */
  int32_t start, end;      /* frames of the keyword's first / last token                */
  int32_t overflow;
  int32_t reserved;
} wekws_ctc_spot_result;
WEKWS_API int64_t wekws_ctc_spot_state_bytes(void);
WEKWS_API int wekws_ctc_spot(const float* d_probs, int V, const int32_t* d_rows, const int32_t* d_frames, int64_t B,
                   const int32_t* d_keyword_tokens, int n_keyword_tokens, const int32_t* d_kw_tokens,
                   const int32_t* d_kw_offsets, int num_keywords, int score_beam_size, int path_beam_size,
                   int frame_stride, double threshold, int min_frames, int max_frames, int interval_frames,
                   void* d_state, void* d_det, wekws_ctc_spot_result* d_result, void* stream);

/* Streaming scoring of a CTC test set (wekws/bin/stream_score_ctc.py:221-377): every utterance b decodes its first
 * d_lens[b] rows of d_probs (B,T,V) frame by frame from the empty hypothesis, with the detection rule of that script
 * (:236-374), quirks included:
 *   - a frame whose top-score_beam_size tokens all fail the filter (prob > 0.05 and in d_keyword_tokens) is skipped
 *     entirely, detection included;
 *   - hit keyword, start, end and hit_score persist across frames and are reset (with the hypotheses) only on
 *     activation, so once a keyword has been seen only the first hypothesis is searched and hit_score = sqrt(hit_score)
 *     runs on every later decoded frame; the stale start / end are tested again;
 *   - activation needs hit_score >= threshold and min_frames <= end - start <= max_frames (no interval rule) and does
 *     not end the utterance; decoding goes on and can activate again.
 * Frame numbers are t * frame_stride (frame_skip), from 0 in each utterance.
 *   d_keyword_tokens: {0} + every keyword token; d_kw_tokens / d_kw_offsets: the keywords in --keywords order, as in
 *   wekws_ctc_spot.
 * Outputs: d_count[b] = activations of utterance b (all of them, even past capacity); d_detections[b * max_detections
 * + i], i < min(count, max_detections), the activations in firing order; d_overflow[b] != 0 if a prefix outgrew
 * WEKWS_CTC_MAX_PREFIX tokens.  A caller that finds a count above max_detections launches again with more room:
 * decoding is deterministic, so the second launch gives the same records.  d_detections may be NULL when
 * max_detections is 0.                                                                                          */
typedef struct {
  double score;            /* hit_score at activation                                   */
  int32_t keyword;         /* index into the keyword list                               */
  int32_t start, end;      /* frames of the keyword's first / last token                */
  int32_t frame;           /* t * frame_stride of the frame that activated              */
} wekws_ctc_stream_detection;
WEKWS_API int wekws_ctc_stream_score(const float* d_probs, const int32_t* d_lens, int64_t B, int64_t T, int V,
                           const int32_t* d_keyword_tokens, int n_keyword_tokens, const int32_t* d_kw_tokens,
                           const int32_t* d_kw_offsets, int num_keywords, int score_beam_size, int path_beam_size,
                           int frame_stride, double threshold, int min_frames, int max_frames, int max_detections,
                           int32_t* d_count, wekws_ctc_stream_detection* d_detections, int32_t* d_overflow,
                           void* stream);

/* Streaming front-end state of KeyWordSpotter.accept_wave (wekws/bin/stream_kws_ctc.py:335-398), B streams.
 *
 * wekws_stream_pcm (:346-364, the wave_remained bookkeeping): stream b appends d_chunk_len[b] int16 samples of row b
 * of d_chunk (0 = no new audio) to its remainder of d_rem_len[b] samples (row b of d_remainder, rem_stride samples per
 * row), writes remainder || chunk to row b of d_stage (stage_stride samples per row; the input of wekws_fbank_forward
 * with per-stream lengths) and keeps stage[d_consumed[b] .. d_rem_len[b] + d_chunk_len[b]) as its new remainder
 * (d_consumed = frames * frame_shift, or 0 while the stream holds its audio).  The caller tracks the lengths.
 *
 * wekws_stream_context (:366-397, context expansion with the carried feature remainder and frame skip): stream b has
 * d_nfeat[b] raw feature rows (row width D) at row b of d_feats (feat_stride rows per stream); 0 = no new features,
 * the stream is not touched.  Its padded sequence is [first row x left] || feats when d_rem_rows[b] == 0 (first chunk)
 * and remainder[0 .. d_rem_rows[b]) || feats otherwise; context row c is the concatenation of padded rows
 * c .. c + left + right.  Output row j (j < d_nout[b]) is context row d_skip_off[b] + j * skip, written to row
 * d_dst_row[b] + j of d_out (row width D * (left + right + 1)).  Then the last min(left + right, nfeat) raw rows become
 * the stream's remainder (row b of d_remainder, (left + right) x D floats per stream).  left = right = 0: no context
 * expansion, the rows are copied (frame skip only).  Values are copied, never computed.  d_out may be NULL only
 * if every d_nout[b] is 0.                                                                                        */
WEKWS_API int wekws_stream_pcm(const int16_t* d_chunk, int64_t chunk_stride, int64_t B, const int32_t* d_chunk_len,
                     const int32_t* d_rem_len, const int32_t* d_consumed, int16_t* d_remainder, int64_t rem_stride,
                     int16_t* d_stage, int64_t stage_stride, void* stream);
WEKWS_API int wekws_stream_context(const float* d_feats, int64_t feat_stride, int64_t B, int D, const int32_t* d_nfeat,
                         const int32_t* d_rem_rows, const int32_t* d_skip_off, const int32_t* d_nout,
                         const int32_t* d_dst_row, int left, int right, int skip, float* d_remainder, float* d_out,
                         void* stream);

/* Context expansion + frame skipping of the FSMN / CTC recipes (SURVEY 8f-4): wekws/dataset/processor.py:267-312
 * (batched twin wekws/dataset/init_dataset.py:24-68).  d_feats (B,T,D); d_lens NULL = all T frames valid;
 * d_out (B, out_frames, D*(left+right+1)): row i of stream b = concat(feats[max(i*skip+k-left, 0)], k = 0..left+right)
 * for i < wekws_context_expand_frames(lens[b], right, skip), zeros after.                                      */
WEKWS_API int64_t wekws_context_expand_frames(int64_t num_frames, int right, int skip);
WEKWS_API int wekws_context_expand(const float* d_feats, const int32_t* d_lens, int64_t B, int64_t T, int D, int left,
                         int right, int skip, float* d_out, int64_t out_frames, void* stream);

/* Raw PCM -> posteriors: Fbank(+CMVN from the model's global_cmvn.* if set) -> model.
 * d_feat_scratch: (B, frames, idim) floats of workspace owned by the caller.  d_out as wekws_model_forward:
 * (B, frames, odim), or (B, odim) with a GLOBAL / LAST head.                          */
WEKWS_API int wekws_pipeline_forward(wekws_fbank* fb, wekws_model* m, const void* d_pcm, int pcm_dtype,
                           int64_t B, int64_t num_samples, int64_t pcm_stride,
                           float* d_feat_scratch, const float* d_in_cache, float* d_out,
                           float* d_out_cache, uint32_t flags, void* stream);

/* Held-out loss and accuracy with the training criteria of wekws/model/loss.py criterion() (as
 * wekws/utils/executor.py Executor.cv / Executor.test call it).  Each call writes d_loss (one float: the criterion's
 * loss) and d_acc (one double: its accuracy) and, when the pointers are not NULL, per-term losses and per-utterance
 * counts.  d_workspace: the bytes the matching *_workspace_bytes query returns, owned by the caller.
 *
 * wekws_criterion_max_pooling (loss.py:26-88): d_logits (B,T,D) posteriors, d_target (B) (< 0 = filler, >= D = no
 *   keyword column), d_lens (B) with max(lens) == T (the caller checks).  Loss: sum of the B*D terms in (i, j) order
 *   in float32, / B.  d_acc = correct / B.  d_term_loss (B,D); d_correct (B) 0/1.  2 launches.
 * wekws_criterion_ce (loss.py:91-100,167-180): d_logits (B,C), d_target (B) in 0..C-1 or -100 (ignored: no term, not
 *   counted; the caller checks the range).  Loss: mean over the counted rows; d_acc = 100 * (argmax == target) / B.
 *   d_utt_loss (B); d_correct (B) 0/1.  2 launches.
 * wekws_criterion_ctc (loss.py:102-164): d_logits (B,T,V) logits, d_lens (B) in 0..T.  Label b is
 *   d_labels[b * label_stride ...] (padded layout) or, with label_stride == 0, the labels back to back (F.ctc_loss's
 *   1-D layout); d_label_lens (B); every label <= max_label_len <= WEKWS_CRITERION_MAX_LABEL tokens, each in 0..V-1
 *   (the caller checks).  Loss: sum of the per-utterance CTC losses (blank 0, +inf for an infeasible utterance) / B.
 *   validation != 0: d_acc = 100 * sum_b (L_b - edit distance of the best prefix-beam hypothesis (score beam 3, path
 *   beam 5) to label b) / sum_b L_b over non-empty labels (NaN when every label is empty), d_overflow (B) != 0 if
 *   utterance b's decode outgrew WEKWS_CTC_MAX_PREFIX tokens (its count is then not the reference's), d_correct (B)
 *   = L_b - distance, d_best (B, 1 + WEKWS_CTC_MAX_PREFIX) = the best hypothesis' length, then its tokens (-1
 *   padded).  validation == 0: d_acc = 0.  d_utt_loss (B).  3 launches, 5 with validation.                      */
#define WEKWS_CRITERION_MAX_LABEL 511
WEKWS_API int64_t wekws_criterion_max_pooling_workspace_bytes(int64_t B, int D);
WEKWS_API int wekws_criterion_max_pooling(const float* d_logits, const int32_t* d_target, const int32_t* d_lens,
                                int64_t B, int64_t T, int D, int min_duration, void* d_workspace, float* d_loss,
                                double* d_acc, float* d_term_loss, int32_t* d_correct, void* stream);
WEKWS_API int64_t wekws_criterion_ce_workspace_bytes(int64_t B);
WEKWS_API int wekws_criterion_ce(const float* d_logits, const int32_t* d_target, int64_t B, int C, void* d_workspace,
                       float* d_loss, double* d_acc, float* d_utt_loss, int32_t* d_correct, void* stream);
WEKWS_API int64_t wekws_criterion_ctc_workspace_bytes(int64_t B, int64_t T, int validation);
WEKWS_API int wekws_criterion_ctc(const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                        const int32_t* d_labels, int64_t label_stride, const int32_t* d_label_lens, int max_label_len,
                        int validation, void* d_workspace, float* d_loss, double* d_acc, float* d_utt_loss,
                        int32_t* d_correct, int32_t* d_overflow, int32_t* d_best, void* stream);

/* Resampling: torchaudio.transforms.Resample(orig_freq, new_freq) with sinc_interp_hann (the resampling of
 * wekws/dataset/processor.py resample() and tools/compute_cmvn_stats.py:50-53), for B waveforms of their own lengths.
 * h_kernel: the (new/g, 2*width + orig/g) float32 table of torchaudio's _get_sinc_resample_kernel (g = gcd of the
 * rates) and its width.  The handle keeps each phase's non-zero span in shared memory; create refuses a rate pair
 * whose compact table does not fit (WEKWS_ERR_INVALID, the message states the size).  Equal rates are refused too:
 * the transform returns its input unchanged.
 * wekws_resample_output_length = ceil(new * n / orig) (0 for n = 0).
 * wekws_resample_forward: d_pcm as wekws_fbank_forward (int16 or float32 at int16 scale, row b at b * pcm_stride
 * elements); d_lens optional (NULL = num_samples each; samples at or past lens[b] count as zeros, they are never
 * read as data).  Row b of d_out (out_stride floats per row) gets the resampling of its first lens[b] samples,
 * accumulated in double and rounded once to float32, then zeros up to max_out, which must be at least
 * wekws_resample_output_length(num_samples).  One launch.                                                      */
typedef struct wekws_resample wekws_resample;
WEKWS_API int wekws_resample_create(int orig_freq, int new_freq, const float* h_kernel, int width,
                                    wekws_resample** out);
WEKWS_API void wekws_resample_destroy(wekws_resample* h);
WEKWS_API int64_t wekws_resample_output_length(const wekws_resample* h, int64_t num_samples);
WEKWS_API int wekws_resample_forward(wekws_resample* h, const void* d_pcm, int pcm_dtype, int64_t B,
                                     int64_t num_samples, int64_t pcm_stride, const int32_t* d_lens, float* d_out,
                                     int64_t out_stride, int64_t max_out, void* stream);

/* Global CMVN statistics (tools/compute_cmvn_stats.py): adds the first d_frames[b] rows of every utterance of
 * d_feats (B, max_frames, D) to d_acc = double[2][D] (sum x, then sum x^2, per dimension) and their count to
 * *d_frame_num.  Per-utterance sums are formed in double in a fixed order and folded into d_acc in utterance order,
 * so the result depends on the order of the utterances only, not on how they are split into calls.
 * d_workspace: wekws_cmvn_stats_workspace_bytes(B, D) bytes owned by the caller.  Two launches.                 */
WEKWS_API int64_t wekws_cmvn_stats_workspace_bytes(int64_t B, int D);
WEKWS_API int wekws_cmvn_stats_accumulate(const float* d_feats, int64_t B, int64_t max_frames, int D,
                                          const int32_t* d_frames, double* d_acc, int64_t* d_frame_num,
                                          void* d_workspace, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* WEKWS_B200_H_ */
