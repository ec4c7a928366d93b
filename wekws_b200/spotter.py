"""Online CTC keyword spotting for many live audio streams, every piece of state on the device.

The batched twin of the reference's one online detector, ``KeyWordSpotter`` (wekws/bin/stream_kws_ctc.py:218-529):
each call takes one chunk of int16 PCM per stream and returns, per stream, exactly what ``KeyWordSpotter.forward``
returns for that chunk -- ``{}`` or ``{state, keyword, start, end, score}`` -- with the reference's rules and quirks
(the 800-sample hold with context expansion, the carried context remainder and frame-skip offset, ``hit_score`` carried
across frames, the reset-and-skip on activation, the end-of-chunk ``max_frames`` reset).

Per call: stream_pcm_kernel (PCM remainder) -> Fbank -> stream_context_kernel (context remainder, frame skip) -> the
model with the fused softmax, once per group of streams with the same frame count -> ctc_spot_kernel (beam search +
detection).  The host keeps an integer mirror of every count (remainder lengths, context rows, skip offset), so it
knows each stream's frame count before anything runs and never reads state back; the only device-to-host copy per
call is the result.

One deliberate difference: the reference raises when a buffer yields fewer frames than it needs (no context expansion
and fewer than one window of samples; or right context 1 and one frame), losing those samples.  Here the stream holds
its samples and returns ``{}`` until the buffer is long enough.

``ThresholdSpotter`` is the detector of the max-pooling (Sigmoid) recipes, which the reference has only as an offline
rule: the same front half (StreamFrontEnd), the model's own Sigmoid, then threshold_spot_kernel, which fires where
wekws/bin/compute_det.py:91-97 counts an alarm on the stream's concatenated posteriors.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np
import torch

from . import _native
from .ctc import SPOT_RESULT_DTYPE, CtcSpotDecoder, check_spot_args
from .frontend import Fbank, Mfcc


class StreamMirror:
    """Host copy of every integer in the per-stream state of accept_wave (stream_kws_ctc.py:335-398).

    win / shift: samples per window / hop; left == right: context rows (0 = no context expansion); skip: frame_skip.
    ``advance(lengths)`` consumes one chunk per stream and returns the counts of that chunk (numpy int64 arrays):
    rem_len / ctx_rows / skip_off before the chunk, consumed samples, stage (fbank input) length, raw feature rows
    ``nfeat`` and model frames ``nout``."""

    def __init__(self, num_streams: int, win: int = 400, shift: int = 160, left: int = 0, right: int = 0,
                 skip: int = 1):
        if left != right or left < 0:
            raise ValueError(f"context expansion needs left == right >= 0, got left {left}, right {right}")
        self.B, self.win, self.shift, self.left, self.right, self.skip = num_streams, win, shift, left, right, skip
        # wave.size < frame_length * right holds the audio (stream_kws_ctc.py:348-351); below one window (no context),
        # or with at most `right` frames (the assert of :367), the reference raises -- here the stream holds instead
        self.hold = max(win * right, win + shift * right)
        self.rem_capacity = self.hold - 1
        self.rem_len = np.zeros(num_streams, dtype=np.int64)
        self.ctx_rows = np.zeros(num_streams, dtype=np.int64)     # 0 = feature_remained is None (first chunk)
        self.skip_off = np.zeros(num_streams, dtype=np.int64)

    def reset(self, streams=None) -> None:
        idx = slice(None) if streams is None else np.asarray(list(streams), dtype=np.int64)
        self.rem_len[idx] = 0
        self.ctx_rows[idx] = 0
        self.skip_off[idx] = 0

    def advance(self, lengths) -> Dict[str, np.ndarray]:
        lens = np.asarray(lengths, dtype=np.int64)
        total = self.rem_len + lens
        run = total >= self.hold
        nfeat = np.where(run, 1 + (total - self.win) // self.shift, 0)
        consumed = nfeat * self.shift
        L, R, ds = self.left, self.right, self.skip
        pre = np.where(self.ctx_rows == 0, L, self.ctx_rows)
        nctx = np.where(run, pre + nfeat - 2 * R, 0)          # len(feats_pad) - 2 * right (nfeat without context)
        off = self.skip_off
        nout = np.where(run & (nctx > off), (nctx - off + ds - 1) // ds, 0)
        last_rem = np.where(off == 0, 0, ds - off)            # stream_kws_ctc.py:391-397
        rem = (nctx + last_rem) % ds
        plan = dict(rem_len=self.rem_len.copy(), chunk_len=lens, consumed=consumed,
                    stage_len=np.where(run, total, 0), nfeat=nfeat, ctx_rows=self.ctx_rows.copy(),
                    skip_off=off.copy(), nout=nout)
        self.rem_len = total - consumed
        self.ctx_rows = np.where(run, np.minimum(L + R, nfeat), self.ctx_rows)
        self.skip_off = np.where(run, np.where(rem == 0, 0, ds - rem), off)
        return plan


class SpotResult:
    """One call's results.  ``to_python()``: list of B dicts, each what KeyWordSpotter.forward returned for the chunk.
    Arrays (host): ``frames`` (model frames per stream), ``state``, ``keyword`` (index, -1), ``start`` / ``end``
    (frames), ``score``, ``overflow``."""

    def __init__(self, words, resolution, frames, raw, fbank, nfeat, model_input, dst_row):
        self.words, self.resolution, self.frames = words, resolution, frames
        ran = frames > 0
        self.state = np.where(ran, raw["state"], 0)
        self.keyword = np.where(ran & (self.state == 1), raw["keyword"], -1)
        self.start = np.where(ran, raw["start"], 0)
        self.end = np.where(ran, raw["end"], 0)
        self.score = np.where(ran, raw["score"], 0.0)
        self.overflow = np.where(ran, raw["overflow"], 0)
        self._fbank, self._nfeat, self._x, self._dst = fbank, nfeat, model_input, dst_row

    def to_python(self) -> List[dict]:
        out = []
        for b in range(len(self.frames)):
            if self.frames[b] == 0:
                out.append({})
            elif self.state[b] == 1:
                out.append({"state": 1, "keyword": self.words[int(self.keyword[b])],
                            "start": int(self.start[b]) * self.resolution, "end": int(self.end[b]) * self.resolution,
                            "score": float(self.score[b])})
            else:
                out.append({"state": 0, "keyword": None, "start": None, "end": None, "score": None})
        return out

    def fbank_rows(self, b: int) -> torch.Tensor:
        """Stream b's raw front-end rows of this chunk (kaldi.fbank of remainder + chunk), on the device."""
        n = int(self._nfeat[b])
        return self._fbank[b, :n] if n else torch.zeros(0, 0)

    def model_input(self, b: int) -> torch.Tensor:
        """Stream b's model-input rows of this chunk (what accept_wave returned), on the device."""
        n = int(self.frames[b])
        return self._x[int(self._dst[b]):int(self._dst[b]) + n] if n else torch.zeros(0, 0)


def context_rows(context):
    """(left, right) of a spotter's `context` argument (None = no context expansion)."""
    left, right = (0, 0) if context is None else (int(context[0]), int(context[1]))
    if context is not None and (left != right or left < 1):
        raise ValueError(f"context expansion is supported with left == right >= 1 (every shipped config is 2, 2), "
                         f"got left {left}, right {right}")
    return left, right


def front_end_settings(configs: dict):
    """(frontend, context, frame_skip, frame_shift in seconds) from `dataset_conf` the way KeyWordSpotter.__init__
    reads them (stream_kws_ctc.py:239-260): feature_extraction_conf.{num_mel_bins, frame_length, frame_shift},
    frame_skip (default 1), context_expansion + context_expansion_conf.{left, right}.  The training recipes name the
    feature section `fbank_conf`; it is accepted when `feature_extraction_conf` is absent."""
    ds = configs["dataset_conf"]
    fe = ds["feature_extraction_conf"] if "feature_extraction_conf" in ds else ds["fbank_conf"]
    frontend = Fbank(fe["num_mel_bins"], frame_length=fe["frame_length"], frame_shift=fe["frame_shift"])
    return (frontend, *_context_settings(ds), fe["frame_shift"] / 1000)


def _context_settings(ds: dict):
    """(context, frame_skip) of a `dataset_conf`: context_expansion + context_expansion_conf.{left, right} (None when
    off) and frame_skip (default 1)."""
    context = None
    if ds.get("context_expansion", False):
        context = (ds["context_expansion_conf"]["left"], ds["context_expansion_conf"]["right"])
    return context, ds.get("frame_skip", 1)


def trained_front_end(configs: dict):
    """(frontend, context, frame_skip) of the features a recipe trains its model on, from `dataset_conf`.  The feature
    type is feature_extraction_conf.feature_type (the shipped configs, wekws/dataset/dataset.py:158-163) or feats_type
    with its `{feats_type}_conf` section; a section without a type is Fbank.  'mfcc' is Mfcc(num_ceps, num_mel_bins),
    the front-end of the mdtc / mdtc_small recipes; 'fbank' is Fbank(num_mel_bins).  Both take frame_length /
    frame_shift in ms."""
    ds = configs["dataset_conf"]
    if "feats_type" in ds:
        ftype, fe = ds["feats_type"], ds[f"{ds['feats_type']}_conf"]
    else:
        fe = ds["feature_extraction_conf"] if "feature_extraction_conf" in ds else ds["fbank_conf"]
        ftype = fe.get("feature_type", "fbank")
    kw = dict(frame_length=fe["frame_length"], frame_shift=fe["frame_shift"])
    if ftype == "mfcc":
        frontend = Mfcc(int(fe.get("num_ceps", 80)), int(fe["num_mel_bins"]), **kw)
    elif ftype == "fbank":
        frontend = Fbank(int(fe["num_mel_bins"]), **kw)
    else:
        raise ValueError(f"feature type {ftype!r}: the recipes use 'fbank' or 'mfcc'")
    return (frontend, *_context_settings(ds))


class FrontChunk:
    """What StreamFrontEnd made of one call: host counts ``nfeat`` / ``nout`` (model frames) / ``dst`` (first row of
    each stream in ``x`` and ``probs``), the device tables ``rows`` / ``frames`` (int32 (B,)) and the device tensors
    ``feats`` (raw front-end rows), ``x`` (model input rows) and ``probs`` (model output rows, None when no stream
    has a frame)."""

    def __init__(self, nfeat, nout, dst, rows, frames, feats, x, probs):
        self.nfeat, self.nout, self.dst, self.rows, self.frames = nfeat, nout, dst, rows, frames
        self.feats, self.x, self.probs = feats, x, probs


class StreamFrontEnd:
    """The streaming half every spotter shares, for `num_streams` streams: PCM remainder, Fbank, context remainder and
    frame skip, and the model with its cache, all state on the device.  A call advances the StreamMirror, groups the
    streams by frame count, uploads one pinned table, runs stream_pcm_kernel, the Fbank and stream_context_kernel, and
    then the model once per group with the cache updated in place; `flags` are the model's forward flags."""

    def __init__(self, model, num_streams: int, frontend: Fbank, left: int, right: int, skip: int, owner: str):
        D = frontend.feature_dim
        if D * (left + right + 1) != model.idim:
            raise ValueError(f"the model takes {model.idim} inputs per frame, the front-end gives {D} x "
                             f"{left + right + 1} context rows")
        params = list(model.parameters()) + list(model.buffers())
        self.dev = params[0].device if params else torch.device("cuda")
        if self.dev.type != "cuda":
            raise RuntimeError(f"{owner} runs on CUDA only: move the model to the GPU first (no CPU fallback)")
        self.model, self.frontend = model, frontend
        self.B, self.D, self.left, self.right, self.skip = int(num_streams), D, left, right, int(skip)
        self.mirror = StreamMirror(self.B, frontend.win, frontend.shift, left, right, self.skip)
        self.cache = torch.zeros(model.cache_shape(self.B), dtype=torch.float32, device=self.dev)
        self.pcm_rem = torch.zeros(self.B, (self.mirror.rem_capacity + 7) // 8 * 8, dtype=torch.int16, device=self.dev)
        self.feat_rem = torch.zeros(self.B, max(left + right, 1), D, dtype=torch.float32, device=self.dev)
        self._table = torch.zeros(9, self.B, dtype=torch.int32).pin_memory()
        self._table_sent = None          # event after the last upload of the pinned table

    def reset(self, streams: Optional[Iterable[int]] = None) -> Optional[List[int]]:
        """PCM and context remainders, skip offset and model cache (an empty cache is a zero cache) of these streams
        (None = all).  Returns the stream list (None = all)."""
        idx = None if streams is None else [int(b) for b in streams]
        if idx is not None and any(not 0 <= b < self.B for b in idx):
            raise ValueError(f"stream index out of range 0..{self.B - 1}")
        self.mirror.reset(idx)
        if idx is None:
            self.cache.zero_()
        elif idx:
            self.cache.index_fill_(self.model.cache_batch_dim, torch.tensor(idx, dtype=torch.int64, device=self.dev),
                                   0.0)
        return idx

    def _forward_group(self, x, out, idx, T, flags):
        """The model over the streams `idx` (host list, ascending) with T frames each, cache in place."""
        m = self.model
        if m.training:
            raise RuntimeError("wekws_b200.KWSModel is inference-only: call model.eval() first")
        h = m._prepare(self.dev)
        n = len(idx)
        whole = n == self.B
        if whole:
            cache = self.cache
        else:
            sel = torch.tensor(idx, dtype=torch.int64, device=self.dev)
            cache = self.cache.index_select(m.cache_batch_dim, sel)
        _native.call("wekws_model_forward", h, x, cache, out, cache, n, T, flags, device=self.dev)
        if not whole:
            self.cache.index_copy_(m.cache_batch_dim, sel, cache)

    def __call__(self, pcm: torch.Tensor, lengths, flags: int) -> FrontChunk:
        """pcm (B, N) int16 CUDA: one chunk per stream; lengths: host ints 0..N (None = N for every stream)."""
        if not isinstance(pcm, torch.Tensor) or not pcm.is_cuda or pcm.dtype != torch.int16 or pcm.dim() != 2:
            raise ValueError("pcm must be a (num_streams, N) int16 CUDA tensor")
        if pcm.size(0) != self.B:
            raise ValueError(f"pcm has {pcm.size(0)} streams, the spotter {self.B}")
        if pcm.device != self.dev:
            raise ValueError(f"pcm is on {pcm.device}, the spotter on {self.dev}")
        N = pcm.size(1)
        if lengths is None:
            lens = np.full(self.B, N, dtype=np.int64)
        else:
            if isinstance(lengths, torch.Tensor) and lengths.is_cuda:
                raise ValueError("lengths are host integers (a CUDA tensor would need a device-to-host copy)")
            lens = np.asarray(lengths, dtype=np.int64).reshape(-1)
            if lens.shape != (self.B,) or (lens < 0).any() or (lens > N).any():
                raise ValueError(f"lengths must be {self.B} integers in 0..{N}")
        if pcm.stride(1) != 1:
            pcm = pcm.contiguous()
        plan = self.mirror.advance(lens)
        nfeat, nout = plan["nfeat"], plan["nout"]
        # streams with the same frame count share one model call; the steady state is one group of every stream
        dst = np.zeros(self.B, dtype=np.int64)
        groups, base = [], 0
        for T in sorted(set(nout[nout > 0].tolist())):
            idx = np.nonzero(nout == T)[0]
            dst[idx] = base + np.arange(len(idx)) * T
            groups.append((int(T), idx.tolist(), base))
            base += len(idx) * T
        if self._table_sent is not None:
            self._table_sent.synchronize()           # the previous call's upload has read the pinned table
        tab = self._table.numpy()
        for r, v in enumerate((plan["chunk_len"], plan["rem_len"], plan["consumed"], plan["stage_len"], nfeat,
                               plan["ctx_rows"], plan["skip_off"], nout, dst)):
            tab[r] = v
        d = self._table.to(self.dev, non_blocking=True)
        self._table_sent = torch.cuda.Event()
        self._table_sent.record(torch.cuda.current_stream(self.dev))
        S = (self.pcm_rem.size(1) + N + 7) // 8 * 8
        stage = torch.empty(self.B, S, dtype=torch.int16, device=self.dev)
        _native.call("wekws_stream_pcm", pcm, pcm.stride(0), self.B, d[0], d[1], d[2], self.pcm_rem,
                     self.pcm_rem.size(1), stage, S, device=self.dev)
        Fmax = int(nfeat.max()) if self.B else 0
        feats = torch.empty(self.B, Fmax, self.D, dtype=torch.float32, device=self.dev)
        x = torch.empty(base, self.model.idim, dtype=torch.float32, device=self.dev)
        if Fmax > 0:
            # the int16 stage rows (remainder + chunk) of each stream through the front-end
            _native.call("wekws_fbank_forward", self.frontend._handle(self.dev), stage, _native.PCM_S16, self.B, S, S,
                         d[3], None, None, feats, Fmax, device=self.dev)
            _native.call("wekws_stream_context", feats, Fmax, self.B, self.D, d[4], d[5], d[6], d[7], d[8], self.left,
                         self.right, self.skip, self.feat_rem, x, device=self.dev)
        probs = None
        if base > 0:
            probs = torch.empty(base, self.model.odim, dtype=torch.float32, device=self.dev)
            for T, idx, row in groups:
                n = len(idx) * T
                self._forward_group(x[row:row + n], probs[row:row + n], idx, T, flags)
        return FrontChunk(nfeat, nout, dst, d[8], d[7], feats, x, probs)


class KeywordSpotter:
    """``KeyWordSpotter`` (stream_kws_ctc.py:218-529) for `num_streams` independent streams, one call per chunk.

        spot = KeywordSpotter(model, {"hi_xiaowen": [5, 9, 17, 23]}, num_streams=B, frontend=Fbank(80),
                              context=(2, 2), frame_skip=3)
        res = spot(pcm)              # pcm (B, N) int16 CUDA, lengths: optional host ints 0..N per stream
        res.to_python()              # [KeyWordSpotter.forward(chunk) for each stream]
        spot.reset([3, 7])           # reset_all() of streams 3 and 7

    `model` is a per-frame KWSModel (CTC: FSMN, DS-TCN, ...) on a CUDA device; its softmax runs fused in the model
    kernel.  Keywords are token-id sequences, in the order the detection tries them."""

    def __init__(self, model, keywords: Dict[str, Sequence[int]], num_streams: int, frontend: Optional[Fbank] = None,
                 context=None, frame_skip: int = 1, threshold: float = 0.0, min_frames: int = 5,
                 max_frames: int = 250, interval_frames: int = 50, score_beam_size: int = 3,
                 path_beam_size: int = 20, resolution: Optional[float] = None):
        if getattr(model, "head", None) is not None:
            raise ValueError(f"KeywordSpotter needs a per-frame model; the '{model.head}' classifier head outputs one "
                             "row per call")
        frontend = frontend if frontend is not None else Fbank(80)
        left, right = context_rows(context)
        check_spot_args(keywords, score_beam_size, path_beam_size, frame_skip)
        if max(t for s in keywords.values() for t in s) >= model.odim:
            raise ValueError(f"a keyword token is outside the model's {model.odim} outputs")
        self.front = StreamFrontEnd(model, num_streams, frontend, left, right, frame_skip, "KeywordSpotter")
        self.dev, self.B = self.front.dev, self.front.B
        # KeyWordSpotter.resolution = frame_shift (ms) / 1000
        self.resolution = frontend.shift * 1000 / int(frontend.cfg.sample_rate) / 1000 if resolution is None else resolution
        self.decoder = CtcSpotDecoder(self.B, keywords, score_beam_size, path_beam_size, self.front.skip, threshold,
                                      min_frames, max_frames, interval_frames, self.dev)
        self.words = self.decoder.words

    @classmethod
    def from_config(cls, configs: dict, model, keywords: Dict[str, Sequence[int]], num_streams: int, **kw):
        """Front-end settings from `dataset_conf` the way KeyWordSpotter.__init__ reads them (front_end_settings)."""
        frontend, context, frame_skip, shift = front_end_settings(configs)
        return cls(model, keywords, num_streams, frontend=frontend, context=context, frame_skip=frame_skip,
                   resolution=shift, **kw)

    @property
    def model(self):
        return self.front.model

    @property
    def frontend(self) -> Fbank:
        return self.front.frontend

    @property
    def cache(self) -> torch.Tensor:
        """Every stream's model cache, on the device (updated in place by each call)."""
        return self.front.cache

    @property
    def mirror(self) -> StreamMirror:
        return self.front.mirror

    def reset(self, streams: Optional[Iterable[int]] = None) -> None:
        """KeyWordSpotter.reset_all() for these streams (None = all): PCM and context remainders, skip offset, model
        cache (an empty cache is a zero cache), hypotheses, hit_score, total_frames, last_active_pos."""
        self.decoder.reset(self.front.reset(streams))

    def __call__(self, pcm: torch.Tensor, lengths=None) -> SpotResult:
        """pcm (B, N) int16 CUDA: one chunk per stream; lengths: host ints 0..N (None = N for every stream)."""
        c = self.front(pcm, lengths, _native.FWD_SOFTMAX)
        raw = np.zeros(self.B, dtype=SPOT_RESULT_DTYPE)
        if c.probs is not None:
            res = self.decoder(c.probs, c.rows, c.frames, live=(c.nout > 0).tolist())
            raw = res.cpu().numpy().view(SPOT_RESULT_DTYPE).reshape(self.B)
        return SpotResult(self.words, self.resolution, c.nout, raw, c.feats, c.nfeat, c.x, c.dst)


def check_rule(thresholds: Sequence[float], window_shift: int) -> List[float]:
    """Validates the alarm rule's arguments; returns the thresholds as floats."""
    thr = [float(t) for t in thresholds]
    if not thr:
        raise ValueError("at least one threshold is needed")
    if not all(np.isfinite(thr)):
        raise ValueError(f"thresholds must be finite, got {thr}")
    if int(window_shift) < 1:
        raise ValueError(f"window_shift must be >= 1, got {window_shift}")
    return thr


def event_slots(max_frames: int, window_shift: int) -> int:
    """Event slots per (stream, keyword) that hold every firing of a call of at most `max_frames` frames: a pair
    fires at most once per `window_shift` frames."""
    return -(-int(max_frames) // int(window_shift)) if max_frames > 0 else 0


class ThresholdDecoder:
    """The alarm rule of wekws/bin/compute_det.py:91-97 online, for `num_streams` streams and K keywords: a frame whose
    6-decimal score reaches the keyword's threshold fires, and the next `window_shift` frames of that stream and
    keyword may not fire.  Each (stream, keyword) record (frames seen, first frame that may fire) stays on the device,
    so over any chunking a stream fires exactly where compute_det.py counts an alarm.  ``__call__`` runs
    threshold_spot_kernel once."""

    def __init__(self, num_streams: int, thresholds: Sequence[float], window_shift: int = 50, device="cuda"):
        thr = check_rule(thresholds, window_shift)
        self.B, self.K, self.window_shift = int(num_streams), len(thr), int(window_shift)
        self.dev = torch.device(device)
        self.thresholds = torch.tensor(thr, dtype=torch.float64, device=self.dev)
        self.state = torch.zeros(self.B, self.K, int(_native.lib().wekws_threshold_spot_state_bytes()),
                                 dtype=torch.uint8, device=self.dev)

    def reset(self, streams: Optional[Iterable[int]] = None) -> None:
        """Restarts these streams (None = all): frame 0 comes next and may fire."""
        if streams is None:
            self.state.zero_()
            return
        idx = [int(b) for b in streams]
        if idx:
            self.state.index_fill_(0, torch.tensor(idx, dtype=torch.int64, device=self.dev), 0)

    def _counts_bytes(self) -> int:
        return (self.B * self.K * 4 + 15) // 16 * 16

    def __call__(self, probs: torch.Tensor, rows: torch.Tensor, frames: torch.Tensor,
                 max_frames: Optional[int] = None) -> torch.Tensor:
        """probs (R, K) float32 CUDA Sigmoid rows, R >= 1; stream b's frames of this call are rows rows[b] .. rows[b] +
        frames[b] - 1 (int32 (B,) tensors on the decoder's device; frames <= 0 = stream untouched).  Without
        `max_frames` the tables are read back and checked against R, and E comes from them.  A caller that passes
        `max_frames` (its host copy of max(frames), as ThresholdSpotter does) vouches for the tables; a value below
        the true maximum makes ``unpack`` raise.  Returns this call's device byte buffer, counts (B, K) int32 then event
        slots (B, K, E) with E = ceil(max_frames / window_shift); ``unpack`` splits it."""
        if (not probs.is_cuda or probs.device != self.dev or probs.dtype != torch.float32 or probs.dim() != 2
                or not probs.is_contiguous() or probs.size(0) == 0):
            raise ValueError(f"probs must be a contiguous (rows >= 1, K) float32 tensor on {self.dev}")
        if probs.size(1) != self.K:
            raise ValueError(f"probs has {probs.size(1)} outputs per row, the decoder {self.K} thresholds")
        for name, t in (("rows", rows), ("frames", frames)):
            if (not isinstance(t, torch.Tensor) or t.device != self.dev or t.dtype != torch.int32
                    or tuple(t.shape) != (self.B,) or not t.is_contiguous()):
                raise ValueError(f"{name} must be a contiguous ({self.B},) int32 tensor on {self.dev}")
        if max_frames is None:
            r, n = torch.stack([rows, frames]).cpu().numpy().astype(np.int64)
            live = n > 0
            if ((r[live] < 0) | (r[live] + n[live] > probs.size(0))).any():
                raise ValueError(f"rows[b] .. rows[b] + frames[b] - 1 must lie in the {probs.size(0)} rows of probs")
            max_frames = int(n.max()) if self.B else 0
        E = event_slots(max_frames, self.window_shift)
        off = self._counts_bytes()
        buf = torch.empty(off + self.B * self.K * E * _native.THRESHOLD_EVENT_BYTES, dtype=torch.uint8,
                          device=self.dev)
        _native.call("wekws_threshold_spot", probs, self.K, rows, frames, self.B, self.thresholds, self.window_shift,
                     self.state, E, buf, buf[off:] if E else None, device=self.dev)
        return buf

    def unpack(self, buf):
        """(counts (B, K) int32, events (B, K, E) records (THRESHOLD_EVENT_DTYPE: frame, keyword, score)) of a
        buffer ``__call__`` returned, as numpy arrays (a CUDA buffer is copied to the host first)."""
        raw = buf.cpu().numpy() if isinstance(buf, torch.Tensor) else np.asarray(buf)
        off, n = self._counts_bytes(), self.B * self.K
        counts = raw[:n * 4].view("<i4").reshape(self.B, self.K)
        E = (raw.size - off) // (n * _native.THRESHOLD_EVENT_BYTES) if n else 0
        events = raw[off:].view(_native.THRESHOLD_EVENT_DTYPE).reshape(self.B, self.K, E)
        if n and int(counts.max()) > E:
            raise RuntimeError(f"a stream fired {int(counts.max())} times in a call with {E} event slots: max_frames "
                               "was below the largest frames[b], so events were not stored")
        return counts, events


class ThresholdResult:
    """One call's results.  Host arrays from one device-to-host copy: ``counts`` (B, K) firings of this call,
    ``events`` (B, K, E) records (frame, keyword, score), the first counts[b, k] of each row valid; ``frames``: model
    frames per stream this call.  ``to_python()``: per stream its firings in frame order."""

    def __init__(self, words, frame_seconds, frames, counts, events, probs, dst, dev):
        self.words, self.frame_seconds, self.frames = words, frame_seconds, frames
        self.counts, self.events = counts, events
        self._probs, self._dst, self._dev = probs, dst, dev

    def to_python(self) -> List[List[dict]]:
        out = []
        for b in range(len(self.frames)):
            evs = [e for k in range(self.counts.shape[1]) for e in self.events[b, k, :self.counts[b, k]]]
            evs.sort(key=lambda e: (int(e["frame"]), int(e["keyword"])))
            out.append([{"keyword": self.words[int(e["keyword"])], "frame": int(e["frame"]),
                         "time": int(e["frame"]) * self.frame_seconds, "score": float(e["score"])} for e in evs])
        return out

    def posteriors(self, b: int) -> torch.Tensor:
        """Stream b's posteriors of this chunk (frames[b], K), on the device (a view, no copy)."""
        n = int(self.frames[b])
        if n == 0:
            return torch.zeros(0, self.counts.shape[1], device=self._dev)
        return self._probs[int(self._dst[b]):int(self._dst[b]) + n]


class ThresholdSpotter:
    """Online keyword spotting with a max-pooling (Sigmoid) model for `num_streams` independent streams, one call per
    chunk, firing by the rule the recipes' DET curves count (compute_det.py:91-97, see ThresholdDecoder).

        spot = ThresholdSpotter(model, thresholds=[0.62, 0.55], num_streams=B, frontend=Fbank(40), window_shift=50,
                                keywords=["HI_XIAOWEN", "NIHAO_WENWEN"])
        res = spot(pcm)              # pcm (B, N) int16 CUDA, lengths: optional host ints 0..N per stream
        res.to_python()              # per stream: [{"keyword", "frame", "time", "score"}, ...]
        spot.reset([3, 7])           # remainders, cache and detection records of streams 3 and 7

    `model` is a per-frame KWSModel with its Sigmoid on a CUDA device; one threshold per output.  A chunk's frames
    are those the whole stream's Fbank would give (remainders are carried), so its firings are those of
    compute_det.py on the stream's concatenated posteriors.  Frames count from the stream's last reset; `time` is
    frame x frame_shift x frame_skip seconds."""

    def __init__(self, model, thresholds: Sequence[float], num_streams: int, frontend: Optional[Fbank] = None,
                 window_shift: int = 50, keywords: Optional[Sequence] = None, context=None, frame_skip: int = 1):
        if getattr(model, "head", None) is not None:
            raise ValueError(f"ThresholdSpotter needs a per-frame model; the '{model.head}' classifier head outputs "
                             "one row per call")
        if not isinstance(getattr(model, "activation", None), torch.nn.Sigmoid):
            raise ValueError(f"ThresholdSpotter needs a model with a Sigmoid output (the max-pooling recipes), got "
                             f"{type(getattr(model, 'activation', None)).__name__}; for a CTC model use KeywordSpotter")
        thr = check_rule(thresholds, window_shift)
        if len(thr) != model.odim:
            raise ValueError(f"one threshold per model output is needed: {model.odim}, got {len(thr)}")
        if int(frame_skip) < 1:
            raise ValueError("frame_skip must be >= 1")
        self.words = list(range(model.odim)) if keywords is None else list(keywords)
        if len(self.words) != model.odim:
            raise ValueError(f"one keyword name per model output is needed: {model.odim}, got {len(self.words)}")
        frontend = frontend if frontend is not None else Fbank(40)
        left, right = context_rows(context)
        self.front = StreamFrontEnd(model, num_streams, frontend, left, right, frame_skip, "ThresholdSpotter")
        self.dev, self.B = self.front.dev, self.front.B
        self.frame_seconds = frontend.shift / int(frontend.cfg.sample_rate) * self.front.skip
        self.decoder = ThresholdDecoder(self.B, thr, window_shift, self.dev)

    @classmethod
    def from_config(cls, configs: dict, model, num_streams: int, thresholds: Sequence[float], **kw):
        """The front-end the model was trained on, from `dataset_conf` (trained_front_end): Fbank, or Mfcc for
        `feature_type: mfcc`; context expansion and frame_skip as KeywordSpotter.from_config reads them."""
        frontend, context, frame_skip = trained_front_end(configs)
        return cls(model, thresholds, num_streams, frontend=frontend, context=context, frame_skip=frame_skip, **kw)

    def reset(self, streams: Optional[Iterable[int]] = None) -> None:
        """PCM and context remainders, skip offset, model cache and detection records of these streams (None = all):
        the next chunk is frame 0 of a fresh stream."""
        self.decoder.reset(self.front.reset(streams))

    def __call__(self, pcm: torch.Tensor, lengths=None) -> ThresholdResult:
        """pcm (B, N) int16 CUDA: one chunk per stream; lengths: host ints 0..N (None = N for every stream)."""
        c = self.front(pcm, lengths, 0)
        K = self.decoder.K
        counts = np.zeros((self.B, K), dtype=np.int32)
        events = np.zeros((self.B, K, 0), dtype=_native.THRESHOLD_EVENT_DTYPE)
        if c.probs is not None:
            counts, events = self.decoder.unpack(self.decoder(c.probs, c.rows, c.frames, int(c.nout.max())))
        return ThresholdResult(self.words, self.frame_seconds, c.nout, counts, events, c.probs, c.dst, self.dev)
