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
 *   wekws_det_stats        the threshold sweep of wekws/bin/compute_det.py:76-105 over whole utterances.
 *   wekws_threshold_spot / the alarm rule of that sweep online, for the max-pooling (Sigmoid) models: the
 *   _state_bytes           per-stream records that let many live streams fire exactly as compute_det.py counts,
 *                          chunk by chunk (added within ABI 19: no existing entry point changed).
 */
#ifndef WEKWS_B200_H_
#define WEKWS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WEKWS_B200_ABI_VERSION 19  /* 2: + wekws_fbank_set_mfcc, wekws_fbank_feature_dim, wekws_det_stats; 3: det max_score is double; 4: precision mode 2, wekws_model_uses_tensor_cores_bt; 5: wekws_model_set_head; 6: + wekws_stream_pcm, wekws_stream_context, wekws_ctc_spot, wekws_ctc_spot_state_bytes; 7: + wekws_ctc_stream_score, wekws_ctc_stream_detection; 8: + wekws_criterion_*; 9: + wekws_resample_*, wekws_cmvn_stats_*; 10: + wekws_fbank_forward_dither, wekws_dither_noise, wekws_spec_aug; 11: + wekws_reverb, wekws_add_noise; 12: + wekws_criterion_*_train, wekws_criterion_*_backward; 13: + wekws_fsmn_* (FSMN training); 14: + wekws_mdtc_* (MDTC training); 15: + wekws_tcn_* (TCN / DS-TCN training), wekws_dropout_mask; 16: + wekws_mdtc_head_* (MDTC training with the global / last head); 17: + wekws_gru_* (GRU training); 18: + wekws_grad_clip*, wekws_adam_step* (the optimiser step); 19: one set of training entry points for every model, wekws_train_* and wekws_model_load_params / _train_forward / _backward, in place of the per-model ones */

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

/* Training front-end (the dither of kaldi.fbank / kaldi.mfcc as wekws/dataset/processor.py compute_fbank /
 * compute_mfcc pass it): wekws_fbank_forward with Gaussian noise of standard deviation `dither` added to every
 * frame after framing, before DC removal, pre-emphasis and the window (torchaudio kaldi.py _get_window).  The
 * noise is not torch.randn's but a pure function of (seed, row b, frame f, sample j): normals from
 * Philox4x32-10 (Random123 constants) with counter (j / 4, f, b, 0) and key (seed lo, seed hi), two Box-Muller
 * pairs per call, u = ((word >> 8) + 0.5) 2^-24, r = sqrt(-2 ln u_a), (r cos 2 pi u_b, r sin 2 pi u_b); each
 * within 1e-6 of the float64 formula.  Log-mel or MFCC by the handle's mode.  One launch.
 * wekws_dither_noise (test hook) writes those normals, d_out (B, frames, frame_length) floats, 16-byte aligned. */
WEKWS_API int wekws_fbank_forward_dither(wekws_fbank* fb, const void* d_pcm, int pcm_dtype, int64_t B,
                                         int64_t num_samples, int64_t pcm_stride, const int32_t* d_lens,
                                         const float* d_mean, const float* d_istd, float* d_out,
                                         int64_t max_frames, float dither, uint64_t seed, void* stream);
WEKWS_API int wekws_dither_noise(uint64_t seed, int64_t B, int64_t frames, float* d_out, void* stream);

/* SpecAugment (wekws/dataset/processor.py spec_aug) on d_feats (B, T, D) in place: for row b, frames t <
 * d_frames[b] that fall in one of its num_t_mask frame ranges, and every column of those frames in one of its
 * num_f_mask column ranges, are set to 0.  d_masks: per row, num_t_mask (start, end) frame pairs then num_f_mask
 * (start, end) column pairs, ends exclusive.  No other element is read or written.  One launch.                */
WEKWS_API int wekws_spec_aug(float* d_feats, const int32_t* d_frames, int64_t B, int64_t T, int D,
                             const int32_t* d_masks, int num_t_mask, int num_f_mask, void* stream);

/* Training-audio augmentation (wekws/dataset/processor.py add_reverb / add_noise).  d_pcm as wekws_fbank_forward
 * (int16 or float32 at int16 scale, row b at b * pcm_stride elements), num_samples per row.  d_rows: (B, 3) int32 on
 * the device, per row (length n_b, offset, count); count 0 = the row is not augmented.  Every sample outside the
 * augmented span [0, n_b) of an augmented row, and every sample of the other rows, is the input converted to float32
 * (exact).  One launch each.
 * wekws_reverb: (offset, count) = the row's RIR, d_rir[offset .. offset + count), all count taps (count > 0, not all
 * zero).  d_out[b][i] = sum_{k <= min(i, count - 1)} h[k] x[i - k] for i < n_b, h = rir / sqrt(sum rir^2): the sum of
 * squares in double in a fixed order, the convolution with FP64 FMAs, rounded once to float32 (within 1 ulp of the
 * float64 evaluation).  A RIR longer than the row costs no more than the row.  d_out (out_stride floats per row) must
 * not overlap d_pcm.
 * wekws_add_noise: (offset, count) = the noise segment s = d_noise[offset .. offset + count); the row adds
 * s[i mod count] for i < n_b (count = n_b for a segment cut from a longer clip, the whole clip otherwise, repeated as
 * np.resize does).  gain = 2^15 sqrt(10^((audio_db - noise_db - d_snr[b]) / 10)), audio_db = 10 log10(mean((x
 * 2^-15)^2) + 1e-4), noise_db = 10 log10(mean(s^2) + 1e-4) over the n_b samples added, in double with a fixed
 * summation order, rounded once to float32; d_out[b][i] = x[i] + gain * s[i mod count] as one float32 multiply and
 * one float32 add.  d_out may be d_pcm when the input is float32 with out_stride == pcm_stride.                  */
WEKWS_API int wekws_reverb(const void* d_pcm, int pcm_dtype, int64_t B, int64_t num_samples, int64_t pcm_stride,
                           const int32_t* d_rows, const float* d_rir, float* d_out, int64_t out_stride, void* stream);
WEKWS_API int wekws_add_noise(const void* d_pcm, int pcm_dtype, int64_t B, int64_t num_samples, int64_t pcm_stride,
                              const int32_t* d_rows, const double* d_snr, const float* d_noise, float* d_out,
                              int64_t out_stride, void* stream);

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

/* Online threshold detector of max-pooling keyword models: the trigger rule of wekws_det_stats (compute_det.py:91-97)
 * applied to live streams chunk by chunk.  Per stream b and keyword k a record in d_state holds two int64: `seen`, the
 * model frames consumed since reset, and `next`, the first frame index that may fire (a zero record is a stream after
 * reset).  Stream b's frames of this call are rows d_rows[b] .. d_rows[b] + d_frames[b] - 1 of d_probs (row width K,
 * the model's Sigmoid outputs); frame i of the call is t = seen + i.  It fires when t >= next and
 * rint((double)p * 1e6) / 1e6 >= d_thresholds[k] (the text-rounded comparison of wekws_det_stats), which records the
 * event (t, k, p) and sets next = t + window_shift; afterwards seen += d_frames[b].  Over the concatenation of a
 * stream's chunks this is the compute_det.py scan for any chunking, so a stream's firings at threshold x number
 * exactly wekws_det_stats' triggers at x.
 *   d_counts (B, K): firings of this call (every one, also for streams with d_frames[b] <= 0, which count 0 and whose
 *   records are not touched).  d_events (B, K, max_events): the first max_events firings of (b, k) in frame order.  A
 *   pair fires at most once per window_shift frames, so max_events = ceil(max_b d_frames[b] / window_shift) holds
 *   every firing.  d_events may be NULL when max_events is 0; every other pointer is required (B > 0).  One launch,
 *   one thread per (b, k), no atomics.                                                                             */
typedef struct {
  int64_t frame;           /* t: model frames since the stream's reset                 */
  int32_t keyword;         /* k                                                        */
  float score;             /* the posterior p as the model wrote it                    */
} wekws_threshold_event;
WEKWS_API int64_t wekws_threshold_spot_state_bytes(void);   /* bytes of one (stream, keyword) record */
WEKWS_API int wekws_threshold_spot(const float* d_probs, int K, const int32_t* d_rows, const int32_t* d_frames,
                                   int64_t B, const double* d_thresholds, int window_shift, void* d_state,
                                   int max_events, int32_t* d_counts, wekws_threshold_event* d_events, void* stream);

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

/* The training step of wekws/utils/executor.py Executor.train (criterion(...), then loss.backward()): the gradient
 * of each criterion's loss with respect to its logits, the one torch's autograd gives for loss.py.
 *
 * wekws_criterion_*_train run the forward above (same arguments, outputs, workspace and launches) and also keep what
 * the gradient needs: max_pooling d_pooled (B,D), the pooled value of every (utterance, column); ce d_count (one
 * float), the number of counted rows; ctc d_utt_loss (B, required here), d_row_max and d_row_sum (B*T each: the
 * softmax normaliser of every frame t < lens[b]) and d_alpha (B, T, 2 * max_label_len + 1: alpha of every frame and
 * extended-label state of each utterance; the rest is not written).
 *
 * wekws_criterion_*_backward write d_grad, every element of a tensor shaped like d_logits, = *d_upstream (one float
 * in device memory: d loss_total / d loss) times d loss / d logits.  No atomics: equal inputs give equal bits.
 *   max_pooling: per (utterance, column) term -1 / (pooled * B) at the pooled frame of the keyword column and
 *     +1 / (pooled * B) for the others, split evenly over the frames whose masked, clamped value equals the pooled
 *     value; a tie that is masked (padding, the first min_duration frames of the keyword column) or outside the
 *     clamp's closed interval [1e-8, 1] counts in the split and gets zero.  1 launch.
 *   ce: (softmax - onehot) / count on counted rows, zero on ignored rows.  1 launch.
 *   ctc: (softmax - occupancy) / B on frames t < lens[b] of a feasible utterance, NaN on those of an infeasible one
 *     (d_utt_loss[b] = +inf), zero on frames t >= lens[b].  The first call (alpha_is_occupancy == 0) overwrites
 *     d_alpha with the state occupancies (beta recurrence, 2 launches); a later call on the same forward passes
 *     alpha_is_occupancy != 0 and reuses them (1 launch).  The logits are read once by the gradient kernel and the
 *     gradient is written once; nothing else of B*T*V elements exists.                                            */
WEKWS_API int wekws_criterion_max_pooling_train(const float* d_logits, const int32_t* d_target, const int32_t* d_lens,
                                int64_t B, int64_t T, int D, int min_duration, void* d_workspace, float* d_loss,
                                double* d_acc, float* d_term_loss, int32_t* d_correct, float* d_pooled, void* stream);
WEKWS_API int wekws_criterion_max_pooling_backward(const float* d_logits, const int32_t* d_target,
                                const int32_t* d_lens, int64_t B, int64_t T, int D, int min_duration,
                                const float* d_pooled, const float* d_upstream, float* d_grad, void* stream);
WEKWS_API int wekws_criterion_ce_train(const float* d_logits, const int32_t* d_target, int64_t B, int C,
                       void* d_workspace, float* d_loss, double* d_acc, float* d_utt_loss, int32_t* d_correct,
                       float* d_count, void* stream);
WEKWS_API int wekws_criterion_ce_backward(const float* d_logits, const int32_t* d_target, int64_t B, int C,
                       const float* d_count, const float* d_upstream, float* d_grad, void* stream);
WEKWS_API int wekws_criterion_ctc_train(const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                        const int32_t* d_labels, int64_t label_stride, const int32_t* d_label_lens, int max_label_len,
                        int validation, void* d_workspace, float* d_loss, double* d_acc, float* d_utt_loss,
                        int32_t* d_correct, int32_t* d_overflow, int32_t* d_best, float* d_row_max, float* d_row_sum,
                        float* d_alpha, void* stream);
WEKWS_API int wekws_criterion_ctc_backward(const float* d_logits, const int32_t* d_lens, int64_t B, int64_t T, int V,
                        const int32_t* d_labels, int64_t label_stride, const int32_t* d_label_lens, int max_label_len,
                        const float* d_row_max, const float* d_row_sum, const float* d_utt_loss, float* d_alpha,
                        int alpha_is_occupancy, const float* d_upstream, float* d_grad, void* stream);

/* Training on the device (wekws/utils/executor.py Executor.train): a training-mode forward that keeps what its backward
 * reads, and the backward to every parameter.  Five models train; every entry point below resolves which one from the
 * handle's backbone and head:
 *   MDTC with the per-frame linear classifier, MDTC with the global / last head, TCN / DS-TCN with the per-frame linear
 *   classifier (the BatchNorm models), FSMN, GRU.
 * A TCN / DS-TCN with a head and a model outside a family's limits below are refused (WEKWS_ERR_INVALID, the message
 * says why).
 *
 * Parameters and gradients travel as host arrays of wekws_train_num_params(m) device pointers, each contiguous float32
 * in the parameter's own shape, in the order each family lists below; a backward writes every element of every
 * gradient buffer, with all B * T frames as rows (padding included, as torch does).  Weight and bias gradients are
 * summed over fixed row slices and the slices added in order: no atomics, equal inputs give equal bits.
 *
 * The queries read the config only.  wekws_train_num_params and the launch counts return 0, the sizes a negative
 * status, for a model they do not accept.  wekws_train_saved_floats(m, B, T): the floats of d_saved a forward of B
 * utterances of T frames writes; wekws_train_backward_workspace_bytes(m, B, T): the bytes of the backward's
 * d_workspace; wekws_train_backward_launches(m): the backward's kernel launches.
 *
 * Two calling conventions; a handle of the other one is refused with a message naming its entry points.
 *
 * The BatchNorm models: wekws_train_forward / wekws_train_backward on a handle that only supplies the config
 * (wekws_model_create, plus wekws_model_set_head for a head).  Everything the kernels read travels with the call, so an
 * optimiser step needs no host round trip.
 *   h_params, n: the parameters.  d_cmvn_mean / d_cmvn_istd: global_cmvn.{mean,istd} (idim floats), or both NULL
 *     without CMVN; cfg.norm_var applies.
 *   h_running: 2 N device pointers, running_mean and running_var of each of the model's N BatchNorms in the order
 *     below; h_bn: 2 N host doubles, (momentum, eps) of the same BatchNorms.  Every BatchNorm normalises with the
 *     biased variance of the batch (all B * T frames, padding included) and updates its running statistics,
 *     running_var with the unbiased variance.  The kernel writes them: a packed eval model of the same weights must be
 *     re-made (wekws_model_finalize) to see them.
 *   Dropout: seed, a 64-bit seed, and h_p, n_p host doubles, one probability in [0, 1] per Dropout module; n_p must be
 *     the model's Dropout count (MDTC 0, h_p may be NULL; MDTC with a head 1; TCN / DS-TCN L, one per block).  Each
 *     module applies a mask that is a pure function of the seed: element e is kept iff (word >> 8) >= theta, theta =
 *     ceil(p 2^24) (in double), word = a component of Philox4x32-10(counter, key = (seed lo, seed hi)) (Random123
 *     constants, as the dither; the dither's counters have word 3 = 0, so the streams are disjoint); a kept element is
 *     multiplied by 1.0f / (float)(1 - p), a dropped one is 0 (selected, not multiplied: p = 1 gives exact zeros).  The
 *     backward recomputes the masks from the same seed and h_p.  wekws_dropout_mask (test hook): d_out (B, T, C) bytes,
 *     1 where block `layer` keeps the element, for theta.
 *   wekws_train_forward: B utterances of T frames (B * T >= 2) from empty caches: d_out, d_out_cache (B, hdim,
 *     padding) as the reference's training-mode new_cache.  save != 0: also writes d_saved; save == 0: d_saved may be
 *     NULL, same d_out / d_out_cache / running-statistics bits.  d_workspace: wekws_train_workspace_bytes(m, B, T,
 *     save) bytes; wekws_train_forward_launches(m) launches either way.
 *   wekws_train_backward: from d_feats, the same h_params / CMVN buffers / seed / h_p and d_saved of a save != 0
 *     forward and d_grad_out = d loss / d out (shaped as d_out), writes h_grads (same shapes as h_params).  d_out, the
 *     forward's logits, is read by the TCN / DS-TCN backward only; the others accept NULL.  Batch statistics are
 *     formed in double over 128 fixed row slices.
 *
 * FSMN and GRU: the packed weights of a handle made by wekws_model_create / _set_tensor / _finalize, as
 * wekws_model_forward runs it.
 *   wekws_model_load_params: the handle's packed weights from h_params, on the device (1 launch): the optimiser's
 *     updates reach the kernels without a host round trip.  The CMVN buffers keep what _finalize packed.
 *   wekws_model_train_forward: wekws_model_forward of B utterances of T frames from empty caches, the same d_out /
 *     d_out_cache bits, also writing d_saved.
 *   wekws_model_backward: from d_feats, d_saved (and, GRU only, d_out, the logits) of that forward and d_grad_out =
 *     d loss / d out (B, T, odim), writes the n = wekws_train_num_params(m) gradient buffers h_grads.
 *
 * MDTC (an mdtc.yaml / mdtc_small.yaml model, wekws/model/mdtc.py): hidden_dim 32 or 64, the per-frame linear
 * classifier (no wekws_model_set_head), input_dim <= 128, output_dim <= 16, kernel_size <= 8, at most 25 blocks.
 *   h_params: 4 + 12 L (L = 1 + num_stack * stack_size blocks), named_parameters order:
 *     preprocessing.out.0.{weight,bias}; per block (backbone.preprocessor, then backbone.blocks.{s}.res_blocks.{l}):
 *     conv1.conv.{weight,bias}, conv1.bn.{weight,bias}, conv1.pointwise.{weight,bias}, bn1.{weight,bias},
 *     conv2.{weight,bias}, bn2.{weight,bias}; classifier.linear.{weight,bias}.
 *   BatchNorms: conv1.bn, bn1, bn2 of each block in block order (N = 3 L).
 *   d_out (B, T, odim).  Saved: 12 L hdim + B T hdim (4 L + 2) floats (each BatchNorm's mean and invstd, the
 *   preprocessing output, per block its three pre-BatchNorm tensors and its output, the stack sum).  Forward workspace
 *   48 * 128 hdim + (save ? 0 : 24 B T hdim) bytes, 2 + 3 L launches.  Every batch statistic and weight-gradient sum is
 *   formed in double over 128 fixed row slices.  Backward workspace 32 * 128 hdim + 20 B T hdim + 8 * 128 P bytes, P
 *   the number of weight and bias elements of the preprocessing Linear, the convolutions and the classifier;
 *   3 + 4 L launches.
 *
 * MDTC with the global / last head (examples/speechcommand_v1/s0/conf/mdtc.yaml): the MDTC backbone as above with the
 * utterance-level head of wekws/model/classifier.py in place of the per-frame linear classifier: GlobalClassifier (the
 * mean over all T frames, padding included) or LastClassifier (frame T - 1) around Linear(hdim, 64) -> ReLU ->
 * Dropout(p) -> Linear(64, odim), the Identity activation; within the MDTC limits except output_dim, here 1..4096.
 *   h_params: 6 + 12 L, the MDTC parameters with classifier.classifier.0.{weight,bias} (64, hdim), (64) and
 *     classifier.classifier.3.{weight,bias} (odim, 64), (odim) in place of classifier.linear.{weight,bias}.
 *   BatchNorms: as MDTC.  Dropout (n_p = 1): element (b, j) of the head's ReLU output (B, 64) uses component j % 4 of
 *     counter (j / 4, 0, b, 256): wekws_dropout_mask(seed, B, 1, 64, 255, theta) gives the mask.  Counter word 3 = 256
 *     keeps the stream apart from the dither's (0) and the TCN blocks' (1..8).
 *   d_out (B, odim).  Saved: 12 L hdim + B T hdim (4 L + 2) + B (hdim + 64) floats (MDTC training's, then the pooled
 *   vectors and the head's pre-ReLU hidden vectors).  Forward workspace 48 * 128 hdim + (save ? 0 : 24 B T hdim) bytes,
 *   3 + 3 L launches.  The head's weight gradients are sums over the utterances in utterance order, in double, rounded
 *   once; the backbone's as MDTC.  Backward workspace 32 * 128 hdim + 24 B T hdim + 8 * 128 P + 512 B bytes, P the
 *   number of weight and bias elements of the preprocessing Linear and the convolutions; 4 + 4 L launches.
 *
 * TCN / DS-TCN (a tcn.yaml / ds_tcn.yaml / ds_tcn_ctc.yaml model, wekws/model/tcn.py): the dense (TCN) and
 * depthwise-separable (DS-TCN) backbones, hidden_dim 64 or 256, kernel_size 2..8, 1..8 layers, input_dim <= 128,
 * output_dim <= 4096; the per-frame linear classifier; Sigmoid or Identity activation.
 *   h_params: 4 + P L (P = 4 dense, 8 ds), named_parameters order: preprocessing.out.0.{weight,bias}; per block
 *     backbone.network.{l}.cnn.: 0.{weight,bias} (the dilated conv), 1.{weight,bias} (BatchNorm), ds only:
 *     3.{weight,bias} (pointwise conv), 4.{weight,bias} (BatchNorm); classifier.linear.{weight,bias}.
 *   BatchNorms: cnn.1 [, cnn.4] of each block in block order (N = L or 2 L).  Dropout (n_p = L): element (b, t, c) of
 *     block l's ReLU output uses p_l and component c % 4 of counter (c / 4, t, b, 1 + l).
 *   d_out (B, T, odim).  Saved: 4 N hdim + B T hdim (1 + L (P / 4 + 1)) floats (each BatchNorm's mean and invstd as
 *   doubles, the preprocessing output, per block its pre-BatchNorm tensors and its output).  Forward workspace
 *   32 * 128 hdim + (save ? 0 : 16 B T hdim) bytes, 2 + L (dense) or 2 + 2 L (ds) launches.  Each weight gradient is
 *   formed over Z fixed row ranges (FP32 over 256 rows, double across them), Z = min(64, max(1, B T / 256),
 *   ceil(264 / tiles)) with tiles = ceil(N / 64) ceil((Q + 1) / 64) for an N x Q weight and its bias, the partials
 *   added in order.  Backward workspace 32 * 128 hdim + 16 B T hdim + 8 (sum of Z N (Q + 1) over the weights,
 *   + 128 hdim (K + 1) per ds block) bytes; 4 + 2 L (dense) or 4 + 3 L (ds) launches.
 *
 * FSMN (an fsmn_ctc.yaml model, wekws/model/fsmn.py FSMN): every FSMN config with at most 32 memory taps
 * (left_order + right_order; the backward keeps one register per tap), with the identity activation.  The three entry
 * points refuse a model with more taps before any launch; wekws_model_forward runs it.
 *   h_params: 8 + 5 L, state_dict order (the model's parameters without the CMVN buffers):
 *     backbone.in_linear1.linear.{weight,bias}, backbone.in_linear2.linear.{weight,bias},
 *     per layer l: backbone.fsmn.{l}.0.linear.weight, .1.conv_left.weight, .1.conv_right.weight,
 *     .2.linear.{weight,bias},
 *     backbone.out_linear1.linear.{weight,bias}, backbone.out_linear2.linear.{weight,bias}
 *     (conv_left.weight is (proj, 1, left_order, 1)).
 *   The forward runs wekws_model_forward's launches.  Saved: B * T * (input_affine_dim + linear_dim + L * (2 proj_dim +
 *   linear_dim) + output_affine_dim) floats.  The weight and bias gradients are summed in 32 fixed row slices.
 *   Backward workspace 4 * (32 * (number of parameter elements) + 2 * B * T * max(input_affine_dim, linear_dim,
 *   proj_dim, output_affine_dim)) bytes; 8 + 5 L launches.
 *
 * GRU (examples/hi_xiaowen/s0/conf/gru.yaml, wekws/model/kws_model.py with the GRU backbone: preprocessing Linear +
 * ReLU, torch.nn.GRU, linear classifier): hidden_dim 128, 1..4 layers, input_dim 1..128, the linear classifier, Sigmoid
 * or Identity.
 *   h_params: 4 + 4 L, named_parameters order: preprocessing.out.0.{weight,bias}, per layer k:
 *     backbone.{weight_ih,weight_hh,bias_ih,bias_hh}_l{k}, classifier.linear.{weight,bias}.  wekws_model_load_params
 *     does not update the tensor-core weight image (the training forward does not read it).
 *   The forward is the FP32 kernel of wekws_model_forward (whatever the precision mode), one launch.  Saved:
 *   (1 + 5 L) B T hidden_dim floats, (B T, hidden_dim) row-major blocks with row b T + t:
 *   x0 = ReLU(Linear(CMVN(feats))), then per layer h_t, r, z, n and W_hn h_{t-1} + b_hn.  Per layer one sequential
 *   kernel runs the recurrence backwards in time; the weight gradients are summed in 32 fixed row slices.  Backward
 *   workspace 4 * (32 P + B T (8 hidden_dim + odim)) bytes, P the number of parameter elements; 5 + 4 L launches.   */
WEKWS_API int wekws_train_num_params(const wekws_model* m);
WEKWS_API int64_t wekws_train_saved_floats(const wekws_model* m, int64_t B, int64_t T);
WEKWS_API int64_t wekws_train_backward_workspace_bytes(const wekws_model* m, int64_t B, int64_t T);
WEKWS_API int wekws_train_backward_launches(const wekws_model* m);
WEKWS_API int64_t wekws_train_workspace_bytes(const wekws_model* m, int64_t B, int64_t T, int save);
WEKWS_API int wekws_train_forward_launches(const wekws_model* m);
WEKWS_API int wekws_train_forward(const wekws_model* m, const float* d_feats, const float* const* h_params, int n,
                                  const float* d_cmvn_mean, const float* d_cmvn_istd, float* const* h_running,
                                  const double* h_bn, uint64_t seed, const double* h_p, int n_p, float* d_out,
                                  float* d_out_cache, float* d_saved, int save, void* d_workspace, int64_t B, int64_t T,
                                  void* stream);
WEKWS_API int wekws_train_backward(const wekws_model* m, const float* d_feats, const float* const* h_params, int n,
                                   const float* d_cmvn_mean, const float* d_cmvn_istd, const float* d_saved,
                                   const float* d_out, const float* d_grad_out, uint64_t seed, const double* h_p,
                                   int n_p, int64_t B, int64_t T, float* const* h_grads, void* d_workspace,
                                   void* stream);
WEKWS_API int wekws_model_load_params(wekws_model* m, const float* const* h_params, int n, void* stream);
WEKWS_API int wekws_model_train_forward(wekws_model* m, const float* d_feats, float* d_out, float* d_out_cache,
                                        float* d_saved, int64_t B, int64_t T, void* stream);
WEKWS_API int wekws_model_backward(wekws_model* m, const float* d_feats, const float* d_saved, const float* d_out,
                                   const float* d_grad_out, int64_t B, int64_t T, float* const* h_grads, int n,
                                   void* d_workspace, void* stream);
WEKWS_API int wekws_dropout_mask(uint64_t seed, int64_t B, int64_t T, int64_t C, int layer, uint32_t theta,
                                 uint8_t* d_out, void* stream);

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

/* The training step's optimiser (wekws/utils/executor.py Executor.train: clip_grad_norm_, then optimizer.step() of
 * torch.optim.Adam).  Tensors travel as host arrays of n device pointers to contiguous float32 data and h_numel[i] >= 1
 * elements each, as in the training entry points.  Each launch takes a table of up to 1024 (clip) or 512 (Adam)
 * tensors in its kernel parameters: nothing is uploaded, nothing allocated, nothing synchronised.
 *
 * wekws_grad_clip: torch.nn.utils.clip_grad_norm_(norm_type=2) on the n gradients, in place.  Launch 1: CTA c of
 *   G = min(264, max(1, ceil(E / 2048))) per table (E the total number of elements) writes the double sum of the
 *   squares of elements [c E_k / G, (c + 1) E_k / G) of its table's concatenated gradients (E_k elements).  Launch 2:
 *   every CTA adds all partials in one fixed order, total_norm = (float)sqrt(sum), and
 *     coef = min((1.0f / (total_norm + 1e-6f)) * (float)max_norm, 1.0f)
 *   each operation rounded to float32, as torch's `max_norm / (total_norm + 1e-6)` (Tensor.__rdiv__: reciprocal, then
 *   multiply) and clamp(max=1) round it; a NaN coefficient stays NaN.  Every gradient element g becomes g * coef
 *   (rounded), also when coef == 1; a non-finite norm propagates as in torch (inf: coef 0, NaN where g is inf).
 *   *d_total_norm gets total_norm.  No atomics: equal inputs give equal bits.  max_norm NaN computes the norm only and
 *   leaves the gradients untouched (the check of clip_grad_norm_(error_if_nonfinite=True) before it scales).
 *   d_workspace: wekws_grad_clip_workspace_bytes(n, E) = 8 G ceil(n / 1024) bytes.
 *   wekws_grad_clip_launches(n) = 2 ceil(n / 1024).
 * wekws_adam_step: one step of torch 2.11's _multi_tensor_adam with amsgrad, maximize and capturable off and L2
 *   weight decay, in place on params, exp_avg and exp_avg_sq; the gradients are read only.  The scalars are rounded
 *   to float32 as torch's foreach kernels take them: w = (float)(1 - beta1), b2 = (float)beta2, c2 = (float)(1 - beta2),
 *   e = (float)eps, wd = (float)weight_decay, and per tensor i ss = (float)h_step_size[i], bc = (float)h_bc2_sqrt[i],
 *   where the caller forms, in double, step_size = (lr / (1 - beta1 ** step)) * -1 and bc2_sqrt = (1 - beta2 ** step)
 *   ** 0.5 with the tensor's own step (torch's own expressions).  Per element, fma() one rounding, every other
 *   operation rounded to float32 on its own:
 *     g = weight_decay != 0 ? fma(wd, p, grad) : grad
 *     m = |w| < 0.5 ? fma(w, g - m, m) : fma(-(g - m), 1 - w, g)        (torch's lerp)
 *     v = fma(c2, g * g, v * b2)
 *     p = fma(ss, m / (sqrt(v) / bc + e), p)
 *   wekws_adam_step_launches(n) = ceil(n / 512).                                                                */
WEKWS_API int64_t wekws_grad_clip_workspace_bytes(int n, int64_t total_elems);
WEKWS_API int wekws_grad_clip_launches(int n);
WEKWS_API int wekws_grad_clip(float* const* h_grads, const int64_t* h_numel, int n, double max_norm,
                              float* d_total_norm, void* d_workspace, void* stream);
WEKWS_API int wekws_adam_step_launches(int n);
WEKWS_API int wekws_adam_step(float* const* h_params, const float* const* h_grads, float* const* h_exp_avg,
                              float* const* h_exp_avg_sq, const int64_t* h_numel, const double* h_step_size,
                              const double* h_bc2_sqrt, int n, double beta1, double beta2, double eps,
                              double weight_decay, void* stream);

#ifdef __cplusplus
}
#endif
#endif  /* WEKWS_B200_H_ */
