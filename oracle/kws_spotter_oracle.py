"""CPU restatement of the reference's online CTC keyword spotter, one stream (wekws/bin/stream_kws_ctc.py:218-529,
``KeyWordSpotter``), built from the pieces of kws_oracle: ``fbank``, ``ctc_prefix_beam_search`` with carried
hypotheses and frame numbers, ``is_sublist``.  It states the semantics wekws_b200.KeywordSpotter keeps, including the
one place it differs on purpose: a buffer too short for the reference (it raises) is held instead.

The model is a callable ``step(feats (T, D) float32) -> probs (T, V) float32`` with ``reset()``; it owns its cache.
``fbank(wave (N,) int64 numpy) -> (m, D) float32`` defaults to kws_oracle.fbank.  Pinned by tests/golden/spotter.npz,
made by running the reference's own class (oracle/make_spotter_golden.py)."""
from __future__ import annotations

import math

import numpy as np
import torch

from . import kws_oracle as O


class SpotterOracle:
    def __init__(self, keywords, model_step, num_mel_bins=80, frame_length=25, frame_shift=10, context=None,
                 frame_skip=1, threshold=0.0, min_frames=5, max_frames=250, interval_frames=50, score_beam_size=3,
                 path_beam_size=20, fbank=None):
        self.keywords = {w: list(t) for w, t in keywords.items()}
        self.tokenset = {0}.union(*[set(t) for t in self.keywords.values()])
        self.model_step = model_step
        self.win = frame_length * 16000 // 1000
        self.shift = frame_shift * 16000 // 1000
        self.resolution = frame_shift / 1000
        self.left, self.right = (0, 0) if context is None else context
        self.context = context is not None
        self.ds = frame_skip
        self.threshold, self.min_frames, self.max_frames = threshold, min_frames, max_frames
        self.interval_frames, self.score_beam, self.path_beam = interval_frames, score_beam_size, path_beam_size
        self.fbank = fbank or (lambda w: O.fbank(torch.from_numpy(w.astype(np.float32)), num_mel_bins,
                                                 float(frame_length), float(frame_shift)))
        # the reference holds the audio while wave.size < frame_length(samples) * right; where it would raise instead
        # (fewer samples than one window, or no more than `right` frames), this restatement holds as well
        self.hold = max(self.win * self.right, self.win + self.shift * self.right)
        self.reset_all()

    # ------------------------------------------------------------------ state
    def reset(self):
        self.cur_hyps = [(tuple(), (1.0, 0.0, []))]
        self.activated = False
        self.hit_score = 1.0

    def reset_all(self):
        self.reset()
        self.wave_remained = np.zeros(0, dtype=np.int64)
        self.feature_remained = None
        self.skip_offset = 0
        self.total_frames = 0
        self.last_active_pos = -1
        self.result = {}
        if hasattr(self.model_step, "reset"):
            self.model_step.reset()

    # ------------------------------------------------------------------ front-end
    def accept_wave(self, samples):
        """New int16 samples -> the model-input rows of this chunk, or None while the audio is held."""
        wave = np.concatenate([self.wave_remained, np.asarray(samples, dtype=np.int64)])
        if wave.size < self.hold:
            self.wave_remained = wave
            return None
        feats = self.fbank(wave)
        n = feats.shape[0]
        self.wave_remained = wave[n * self.shift:]
        if self.context:
            L, R = self.left, self.right
            head = feats[:1].expand(L, -1) if self.feature_remained is None else self.feature_remained
            padded = torch.cat([head, feats])
            rows = padded.shape[0] - 2 * R
            feats_ctx = torch.stack([padded[i:i + L + R + 1].reshape(-1) for i in range(rows)])
            self.feature_remained = feats[max(n - (L + R), 0):]
            feats = feats_ctx
        if self.ds > 1:
            carried = 0 if self.skip_offset == 0 else self.ds - self.skip_offset
            left_over = (feats.shape[0] + carried) % self.ds
            feats = feats[self.skip_offset::self.ds]
            self.skip_offset = 0 if left_over == 0 else self.ds - left_over
        return feats

    # ------------------------------------------------------------------ detection
    def _detect(self, frame):
        word, start, end = None, 0, 0
        for prefix, _, nodes in O.hyps_of(self.cur_hyps):
            for w, lab in self.keywords.items():
                off = O.is_sublist(prefix, lab)
                if off != -1:
                    word, start, end = w, nodes[off]['frame'], nodes[off + len(lab) - 1]['frame']
                    for i in range(off, off + len(lab)):
                        self.hit_score *= nodes[i]['prob']
                    break
            if word is not None:
                self.hit_score = math.sqrt(self.hit_score)
                break
        duration = end - start
        if (word is not None and self.hit_score >= self.threshold and self.min_frames <= duration <= self.max_frames
                and (self.last_active_pos == -1 or end - self.last_active_pos >= self.interval_frames)):
            self.activated = True
            self.last_active_pos = end
        on = self.activated
        self.result = {"state": 1 if on else 0, "keyword": word if on else None,
                       "start": start * self.resolution if on else None, "end": end * self.resolution if on else None,
                       "score": self.hit_score if on else None}

    def forward(self, samples, feats=None):
        """One chunk of int16 samples -> the result dict.  `feats`: model-input rows to use instead of accept_wave's
        own (which still runs, for the state and the row count)."""
        got = self.accept_wave(samples)
        if got is None or got.shape[0] < 1:
            return {}
        if feats is not None:
            assert feats.shape[0] == got.shape[0]
            got = feats
        probs = self.model_step(got)
        T = probs.shape[0]
        for t in range(T):
            frame = t * self.ds + self.total_frames
            self.cur_hyps = O.ctc_prefix_beam_search(probs[t:t + 1], self.tokenset, self.score_beam, self.path_beam,
                                                     cur_hyps=self.cur_hyps, frame_offset=frame)
            self._detect(frame)
            if self.activated:
                self.reset()
                break
        self.total_frames += T * self.ds
        top = self.cur_hyps[0] if self.cur_hyps else None
        if top is not None and len(top[0]) > 0 and self.total_frames - int(top[1][2][0]['frame']) > self.max_frames:
            self.reset()
        return self.result
