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
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Optional, Sequence

import numpy as np
import torch

from . import _native
from .ctc import SPOT_RESULT_DTYPE, CtcSpotDecoder, check_spot_args
from .frontend import Fbank


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
        left, right = (0, 0) if context is None else (int(context[0]), int(context[1]))
        if context is not None and (left != right or left < 1):
            raise ValueError(f"context expansion is supported with left == right >= 1 (every shipped config is 2, 2), "
                             f"got left {left}, right {right}")
        check_spot_args(keywords, score_beam_size, path_beam_size, frame_skip)
        if max(t for s in keywords.values() for t in s) >= model.odim:
            raise ValueError(f"a keyword token is outside the model's {model.odim} outputs")
        D = frontend.feature_dim
        if D * (left + right + 1) != model.idim:
            raise ValueError(f"the model takes {model.idim} inputs per frame, the front-end gives {D} x "
                             f"{left + right + 1} context rows")
        params = list(model.parameters()) + list(model.buffers())
        self.dev = params[0].device if params else torch.device("cuda")
        if self.dev.type != "cuda":
            raise RuntimeError("KeywordSpotter runs on CUDA only: move the model to the GPU first (no CPU fallback)")
        self.model, self.frontend = model, frontend
        self.B, self.D, self.left, self.right, self.skip = int(num_streams), D, left, right, int(frame_skip)
        # KeyWordSpotter.resolution = frame_shift (ms) / 1000
        self.resolution = frontend.shift * 1000 / int(frontend.cfg.sample_rate) / 1000 if resolution is None else resolution
        self.mirror = StreamMirror(self.B, frontend.win, frontend.shift, left, right, self.skip)
        self.decoder = CtcSpotDecoder(self.B, keywords, score_beam_size, path_beam_size, self.skip, threshold,
                                      min_frames, max_frames, interval_frames, self.dev)
        self.words = self.decoder.words
        self.cache = torch.zeros(model.cache_shape(self.B), dtype=torch.float32, device=self.dev)
        self.pcm_rem = torch.zeros(self.B, (self.mirror.rem_capacity + 7) // 8 * 8, dtype=torch.int16, device=self.dev)
        self.feat_rem = torch.zeros(self.B, max(left + right, 1), D, dtype=torch.float32, device=self.dev)
        self._table = torch.zeros(9, self.B, dtype=torch.int32).pin_memory()
        self._table_sent = None          # event after the last upload of the pinned table

    @classmethod
    def from_config(cls, configs: dict, model, keywords: Dict[str, Sequence[int]], num_streams: int, **kw):
        """Front-end settings from `dataset_conf` the way KeyWordSpotter.__init__ reads them (stream_kws_ctc.py:239-260):
        feature_extraction_conf.{num_mel_bins, frame_length, frame_shift}, frame_skip (default 1), context_expansion +
        context_expansion_conf.{left, right}.  The training recipes name the feature section `fbank_conf`; it is
        accepted when `feature_extraction_conf` is absent."""
        ds = configs["dataset_conf"]
        fe = ds["feature_extraction_conf"] if "feature_extraction_conf" in ds else ds["fbank_conf"]
        frontend = Fbank(fe["num_mel_bins"], frame_length=fe["frame_length"], frame_shift=fe["frame_shift"])
        context = None
        if ds.get("context_expansion", False):
            context = (ds["context_expansion_conf"]["left"], ds["context_expansion_conf"]["right"])
        return cls(model, keywords, num_streams, frontend=frontend, context=context,
                   frame_skip=ds.get("frame_skip", 1), resolution=fe["frame_shift"] / 1000, **kw)

    def reset(self, streams: Optional[Iterable[int]] = None) -> None:
        """KeyWordSpotter.reset_all() for these streams (None = all): PCM and context remainders, skip offset, model
        cache (an empty cache is a zero cache), hypotheses, hit_score, total_frames, last_active_pos."""
        idx = None if streams is None else [int(b) for b in streams]
        if idx is not None and any(not 0 <= b < self.B for b in idx):
            raise ValueError(f"stream index out of range 0..{self.B - 1}")
        self.mirror.reset(idx)
        self.decoder.reset(idx)
        if idx is None:
            self.cache.zero_()
        elif idx:
            self.cache.index_fill_(self.model.cache_batch_dim, torch.tensor(idx, dtype=torch.int64, device=self.dev),
                                   0.0)

    def _forward_group(self, x, out, idx, T):
        """The model over the streams `idx` (host list, ascending) with T frames each, softmax fused, cache in place."""
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
        _native.call("wekws_model_forward", h, x, cache, out, cache, n, T, _native.FWD_SOFTMAX, device=self.dev)
        if not whole:
            self.cache.index_copy_(m.cache_batch_dim, sel, cache)

    def __call__(self, pcm: torch.Tensor, lengths=None) -> SpotResult:
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
        raw = np.zeros(self.B, dtype=SPOT_RESULT_DTYPE)
        if Fmax > 0:
            # the int16 stage rows (remainder + chunk) of each stream through the front-end
            _native.call("wekws_fbank_forward", self.frontend._handle(self.dev), stage, _native.PCM_S16, self.B, S, S,
                         d[3], None, None, feats, Fmax, device=self.dev)
            _native.call("wekws_stream_context", feats, Fmax, self.B, self.D, d[4], d[5], d[6], d[7], d[8], self.left,
                         self.right, self.skip, self.feat_rem, x, device=self.dev)
        if base > 0:
            probs = torch.empty(base, self.model.odim, dtype=torch.float32, device=self.dev)
            for T, idx, row in groups:
                n = len(idx) * T
                self._forward_group(x[row:row + n], probs[row:row + n], idx, T)
            res = self.decoder(probs, d[8], d[7], live=(nout > 0).tolist())
            raw = res.cpu().numpy().view(SPOT_RESULT_DTYPE).reshape(self.B)
        return SpotResult(self.words, self.resolution, nout, raw, feats, nfeat, x, dst)
