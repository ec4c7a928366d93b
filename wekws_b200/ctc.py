"""CTC prefix beam search and keyword look-up on the GPU (SURVEY 8f-2, CTC models).

Replaces the per-utterance / per-frame pure-Python decoding of the reference -- ``wekws/model/loss.py:206-312``
(``ctc_prefix_beam_search``) as called by ``wekws/bin/score_ctc.py:198-226`` and its streaming twin
``wekws/bin/stream_kws_ctc.py:124-215,400-434``, and the streaming scorer ``wekws/bin/stream_score_ctc.py:221-377``
-- with one kernel over all utterances, bit-exact (hypothesis
order, scores as doubles, node frames / probabilities; see csrc/ctc_decode.cu for the Python semantics it keeps).
"""
from __future__ import annotations

import itertools
from typing import Dict, Iterable, List, Optional, Sequence

import torch

from . import _native
from ._native import CTC_MAX_PATH_BEAM as MAX_PATH_BEAM
from ._native import CTC_MAX_PREFIX as MAX_PREFIX
from ._native import CTC_MAX_SCORE_BEAM as MAX_SCORE_BEAM
from ._native import SPOT_RESULT_BYTES, SPOT_RESULT_DTYPE, STREAM_DETECTION_BYTES, STREAM_DETECTION_DTYPE  # noqa: F401

STREAM_SCORE_CAPACITY = 32         # detection records per utterance of the first launch of stream_score_ctc


def _pack_keywords(seqs: Sequence[Sequence[int]], device):
    """Keyword token lists as the kernels take them: int32 device tensors (tokens back to back, offsets), keyword k
    being tokens[offsets[k]:offsets[k + 1]]."""
    offsets = [0, *itertools.accumulate(len(s) for s in seqs)]
    return (torch.tensor([t for s in seqs for t in s], dtype=torch.int32, device=device),
            torch.tensor(offsets, dtype=torch.int32, device=device))


class CtcHyps:
    """Device-side result of ctc_prefix_beam_search: tensors in beam order (see include/wekws_b200.h)."""

    def __init__(self, B, path_beam, dev):
        self.B, self.path_beam = B, path_beam
        self.nhyp = torch.empty(B, dtype=torch.int32, device=dev)
        self.overflow = torch.empty(B, dtype=torch.int32, device=dev)
        self.hyp_len = torch.empty(B, path_beam, dtype=torch.int32, device=dev)
        self.hyp_tokens = torch.empty(B, path_beam, MAX_PREFIX, dtype=torch.int32, device=dev)
        self.hyp_score = torch.empty(B, path_beam, dtype=torch.float64, device=dev)
        self.node_frame = torch.empty(B, path_beam, MAX_PREFIX, dtype=torch.int32, device=dev)
        self.node_prob = torch.empty(B, path_beam, MAX_PREFIX, dtype=torch.float32, device=dev)

    def to_python(self) -> List[list]:
        """The reference's return value per utterance: [(prefix tuple, pb + pnb, [dict(token, frame, prob), ...]), ...]
        (loss.py:311-312)."""
        nh, ln = self.nhyp.cpu().tolist(), self.hyp_len.cpu().tolist()
        tok, sc = self.hyp_tokens.cpu().tolist(), self.hyp_score.cpu().tolist()
        fr, pr = self.node_frame.cpu().tolist(), self.node_prob.cpu().tolist()
        out = []
        for b in range(self.B):
            hyps = []
            for h in range(nh[b]):
                n = ln[b][h]
                hyps.append((tuple(tok[b][h][:n]), sc[b][h],
                             [dict(token=tok[b][h][i], frame=fr[b][h][i], prob=pr[b][h][i]) for i in range(n)]))
            out.append(hyps)
        return out


def ctc_state(num_streams: int, device) -> torch.Tensor:
    """Opaque per-stream hypothesis state for chunked / streaming decoding (stream_kws_ctc.py keeps `cur_hyps`)."""
    return torch.zeros(num_streams, int(_native.lib().wekws_ctc_state_bytes()), dtype=torch.uint8, device=device)


def ctc_prefix_beam_search(probs: torch.Tensor, lengths: Optional[torch.Tensor] = None,
                           keywords_tokenset: Optional[Iterable[int]] = None, score_beam_size: int = 3,
                           path_beam_size: int = 20, state: Optional[torch.Tensor] = None, reset_state: bool = True,
                           frame_offset: int = 0, frame_stride: int = 1) -> CtcHyps:
    """probs (B, T, V) float32 CUDA softmax posteriors (score_ctc.py:195 `logits.softmax(2)`), lengths (B,).
    With `state` (from ctc_state) the final hypotheses are kept; pass reset_state=False on the following chunks and
    frame_offset = frames decoded so far to continue a stream exactly as stream_kws_ctc.py does frame by frame."""
    if not probs.is_cuda:
        raise RuntimeError("wekws_b200.ctc_prefix_beam_search runs on CUDA only; got a CPU tensor (no CPU fallback)")
    if probs.dim() != 3 or probs.dtype != torch.float32:
        raise ValueError("probs must be a (B, T, V) float32 tensor")
    probs = probs.contiguous()
    B, T, V = probs.shape
    dev = probs.device
    out = CtcHyps(B, path_beam_size, dev)
    lens = None if lengths is None else lengths.to(device=dev, dtype=torch.int32).contiguous()
    kw = None
    if keywords_tokenset is not None:
        kw = torch.tensor(sorted(int(t) for t in keywords_tokenset), dtype=torch.int32, device=dev)
        if kw.numel() == 0:
            raise ValueError("keywords_tokenset is empty (use None for no filter)")
    if state is not None and (state.dtype != torch.uint8 or state.device != dev or not state.is_contiguous()
                              or tuple(state.shape) != (B, int(_native.lib().wekws_ctc_state_bytes()))):
        raise ValueError("state must come from ctc_state(B, device)")
    _native.call("wekws_ctc_prefix_beam_search", probs, lens, B, T, V, kw, 0 if kw is None else kw.numel(),
                 int(score_beam_size), int(path_beam_size), int(frame_offset), int(frame_stride), state,
                 1 if reset_state else 0, out.nhyp, out.hyp_len, out.hyp_tokens, out.hyp_score, out.node_frame,
                 out.node_prob, out.overflow, device=dev)
    return out


def ctc_keyword_hits(hyps: CtcHyps, keywords_token: Dict[str, dict]):
    """score_ctc.py:201-220 on the device: for every utterance the first hypothesis (beam order) that contains a keyword
    (dict order) -> list of (word or None, hit_score, start_frame, end_frame).  keywords_token: {word: {'token_id':
    [...]}} as the reference builds it (score_ctc.py:159-171)."""
    words = list(keywords_token.keys())
    dev = hyps.nhyp.device
    flat, offs = _pack_keywords([list(keywords_token[w]["token_id"]) for w in words], dev)
    hit = torch.empty(hyps.B, dtype=torch.int32, device=dev)
    score = torch.empty(hyps.B, dtype=torch.float64, device=dev)
    start = torch.empty(hyps.B, dtype=torch.int32, device=dev)
    end = torch.empty(hyps.B, dtype=torch.int32, device=dev)
    _native.call("wekws_ctc_keyword_hit", hyps.nhyp, hyps.hyp_len, hyps.hyp_tokens, hyps.node_frame, hyps.node_prob,
                 hyps.B, hyps.path_beam, flat, offs, len(words), hit, score, start, end, device=dev)
    hit, score, start, end = hit.cpu().tolist(), score.cpu().tolist(), start.cpu().tolist(), end.cpu().tolist()
    return [(words[h] if h >= 0 else None, score[b], start[b], end[b]) for b, h in enumerate(hit)]


def write_ctc_scores(fout, keys: Sequence[str], hits) -> None:
    """The score file of score_ctc.py:217-226: '{key} detected {keyword} {score:.3f}' or '{key} rejected'."""
    for key, (word, hit_score, _, _) in zip(keys, hits):
        if word is not None:
            fout.write('{} detected {} {:.3f}\n'.format(key, word, hit_score))
        else:
            fout.write('{} rejected\n'.format(key))


def check_spot_args(keywords: Dict[str, Sequence[int]], score_beam_size: int, path_beam_size: int,
                    frame_stride: int = 1):
    """Validates the spotter's decoding arguments; returns (keyword names, token-id lists)."""
    if not keywords:
        raise ValueError("at least one keyword is needed")
    if not 1 <= int(score_beam_size) <= MAX_SCORE_BEAM:
        raise ValueError(f"score_beam_size must be in 1..{MAX_SCORE_BEAM}, got {score_beam_size}")
    if not 1 <= int(path_beam_size) <= MAX_PATH_BEAM:
        raise ValueError(f"path_beam_size must be in 1..{MAX_PATH_BEAM}, got {path_beam_size}")
    if int(frame_stride) < 1:
        raise ValueError("frame_stride must be >= 1")
    words = list(keywords)
    seqs = [[int(t) for t in keywords[w]] for w in words]
    for w, s in zip(words, seqs):
        if not 1 <= len(s) <= MAX_PREFIX or min(s) < 0:
            raise ValueError(f"keyword {w!r}: 1..{MAX_PREFIX} non-negative token ids are needed, got {s}")
    return words, seqs


class StreamScores:
    """Result of stream_score_ctc.  ``count`` (B,) int32: activations per utterance; ``detections`` (B, capacity, 24)
    uint8: the records in firing order (decode with STREAM_DETECTION_DTYPE); ``overflow`` (B,) int32: != 0 if a
    prefix outgrew MAX_PREFIX tokens (the decode of that utterance is then not the reference's); ``launches``: kernel
    launches the call made (1, or 2 when some utterance activated more than STREAM_SCORE_CAPACITY times)."""

    def __init__(self, words, count, detections, overflow, launches):
        self.words, self.count, self.detections, self.overflow = words, count, detections, overflow
        self.launches = launches

    def to_python(self) -> List[List[tuple]]:
        """Per utterance, its activations [(keyword, score, start, end, frame)] in firing order; frame is
        t * frame_skip of the frame that activated, in the units of start and end."""
        count = self.count.cpu().tolist()
        rec = self.detections.cpu().numpy().view(STREAM_DETECTION_DTYPE)[..., 0]
        return [[(self.words[int(r["keyword"])], float(r["score"]), int(r["start"]), int(r["end"]), int(r["frame"]))
                 for r in rec[b, :n]] for b, n in enumerate(count)]


def stream_score_ctc(probs: torch.Tensor, lengths, keywords: Dict[str, Sequence[int]], score_beam_size: int = 3,
                     path_beam_size: int = 20, threshold: float = 0.0, min_frames: int = 5, max_frames: int = 250,
                     frame_skip: int = 1) -> StreamScores:
    """The frame loop of wekws/bin/stream_score_ctc.py:221-377 over a whole batch, one warp per utterance.

    probs (B, T, V) float32 CUDA softmax posteriors (``model.forward_softmax(feats)`` or ``logits.softmax(2)``);
    lengths (B,) valid frames (``feats_lengths`` after frame skip); keywords {word: token ids} in --keywords order.
    Every activation is kept: a first launch stores STREAM_SCORE_CAPACITY records per utterance and counts them all;
    if some utterance activated more often, one more launch with room for the largest count follows."""
    words, seqs = check_spot_args(keywords, score_beam_size, path_beam_size, frame_skip)
    if not torch.is_tensor(probs) or probs.dim() != 3 or probs.dtype != torch.float32:
        raise ValueError("probs must be a (B, T, V) float32 tensor")
    B, T, V = probs.shape
    lens_host = torch.as_tensor(lengths).detach().cpu()
    if lens_host.numel() == 0:
        lens_host = lens_host.long()
    if lens_host.dtype.is_floating_point or lens_host.dtype == torch.bool or tuple(lens_host.shape) != (B,):
        raise ValueError(f"lengths must be ({B},) integer frame counts")
    if B and (int(lens_host.min()) < 0 or int(lens_host.max()) > T):
        raise ValueError(f"lengths must be in 0..{T} (the frames of probs)")
    tokenset = {0}.union(*[set(s) for s in seqs])
    if max(tokenset) >= V:
        raise ValueError(f"keyword token {max(tokenset)} is outside the vocabulary of {V} outputs")
    if not probs.is_cuda:
        raise RuntimeError("wekws_b200.stream_score_ctc runs on CUDA only; got a CPU tensor (no CPU fallback)")
    dev = probs.device
    probs = probs.contiguous()
    lens = lens_host.to(device=dev, dtype=torch.int32)
    tset = torch.tensor(sorted(tokenset), dtype=torch.int32, device=dev)
    kw, off = _pack_keywords(seqs, dev)
    count = torch.zeros(B, dtype=torch.int32, device=dev)
    overflow = torch.zeros(B, dtype=torch.int32, device=dev)

    def launch(cap):
        det = torch.empty(B, cap, STREAM_DETECTION_BYTES, dtype=torch.uint8, device=dev)
        _native.call("wekws_ctc_stream_score", probs, lens, B, T, V, tset, tset.numel(), kw, off, len(words),
                     int(score_beam_size), int(path_beam_size), int(frame_skip), float(threshold), int(min_frames),
                     int(max_frames), cap, count, det, overflow, device=dev)
        return det

    cap = STREAM_SCORE_CAPACITY
    det = launch(cap)
    launches = 1
    need = int(count.max()) if B else 0
    if need > cap:
        det = launch(need)
        launches = 2
    return StreamScores(words, count, det, overflow, launches)


def write_stream_ctc_scores(fout, keys: Sequence[str], result: StreamScores) -> None:
    """The score file of stream_score_ctc.py:349-376: '{key} detected {keyword} {score:.3f}' per activation, or
    '{key} rejected' for an utterance that never activated."""
    for key, dets in zip(keys, result.to_python()):
        if not dets:
            fout.write('{} rejected\n'.format(key))
        for word, score, _, _, _ in dets:
            fout.write('{} detected {} {:.3f}\n'.format(key, word, score))


class CtcSpotDecoder:
    """The decoding and detection half of the reference's streaming spotter (stream_kws_ctc.py:400-514) for
    `num_streams` streams, with every piece of state on the device: the hypotheses (ctc_state layout), hit_score,
    total_frames and last_active_pos.  ``__call__`` runs ctc_spot_kernel once over every stream with frames."""

    def __init__(self, num_streams: int, keywords: Dict[str, Sequence[int]], score_beam_size: int = 3,
                 path_beam_size: int = 20, frame_stride: int = 1, threshold: float = 0.0, min_frames: int = 5,
                 max_frames: int = 250, interval_frames: int = 50, device="cuda"):
        self.words, seqs = check_spot_args(keywords, score_beam_size, path_beam_size, frame_stride)
        self.B = int(num_streams)
        self.dev = torch.device(device)
        self.score_beam, self.path_beam, self.frame_stride = int(score_beam_size), int(path_beam_size), int(frame_stride)
        self.threshold, self.min_frames = float(threshold), int(min_frames)
        self.max_frames, self.interval_frames = int(max_frames), int(interval_frames)
        tokenset = {0}                                          # set_keywords: keywords_idxset = {0} | every token
        for s in seqs:
            tokenset.update(s)
        self.tokenset = tokenset
        self.max_token = max(tokenset)
        self._set = torch.tensor(sorted(tokenset), dtype=torch.int32, device=self.dev)
        self._kw, self._off = _pack_keywords(seqs, self.dev)
        self.state = ctc_state(self.B, self.dev)
        self.det = torch.zeros(self.B, int(_native.lib().wekws_ctc_spot_state_bytes()), dtype=torch.uint8,
                               device=self.dev)
        self.result = torch.zeros(self.B, SPOT_RESULT_BYTES, dtype=torch.uint8, device=self.dev)
        self._live = [False] * self.B

    def reset(self, streams: Optional[Iterable[int]] = None) -> None:
        """KeyWordSpotter.reset_all() for these streams (None = all): a zero detection record restarts the stream."""
        if streams is None:
            self.det.zero_()
            self._live = [False] * self.B
            return
        idx = [int(b) for b in streams]
        if idx:
            self.det.index_fill_(0, torch.tensor(idx, dtype=torch.int64, device=self.dev), 0)
        for b in idx:
            self._live[b] = False

    def __call__(self, probs: torch.Tensor, rows: torch.Tensor, frames: torch.Tensor,
                 live: Optional[Sequence[bool]] = None) -> torch.Tensor:
        """probs (R, V) float32 CUDA softmax rows; stream b decodes rows rows[b] .. rows[b] + frames[b] - 1 (int32 CUDA
        (B,) tensors; frames 0 = stream untouched).  `live`: host copy of frames > 0, if the caller has it.  Returns
        the (B, 32) byte result buffer (decode with SPOT_RESULT_DTYPE); only streams with frames are written."""
        if not probs.is_cuda or probs.dtype != torch.float32 or probs.dim() != 2 or not probs.is_contiguous():
            raise ValueError("probs must be a contiguous (rows, V) float32 CUDA tensor")
        V = probs.size(1)
        if self.max_token >= V:
            raise ValueError(f"keyword token {self.max_token} is outside the vocabulary of {V} outputs")
        if live is None:
            live = (frames.cpu() > 0).tolist()
        for b, x in enumerate(live):
            if x:
                self._live[b] = True
        _native.call("wekws_ctc_spot", probs, V, rows, frames, self.B, self._set, self._set.numel(), self._kw, self._off,
                     len(self.words), self.score_beam, self.path_beam, self.frame_stride, self.threshold,
                     self.min_frames, self.max_frames, self.interval_frames, self.state, self.det, self.result,
                     device=self.dev)
        return self.result

    def hypotheses(self) -> List[list]:
        """Each stream's carried hypotheses as [(prefix, pb + pnb, nodes)] (hyps_of(cur_hyps))."""
        out = ctc_prefix_beam_search(torch.empty(self.B, 0, 1, device=self.dev), None, None, 1, self.path_beam,
                                     state=self.state, reset_state=False).to_python()
        return [out[b] if self._live[b] else [(tuple(), 1.0, [])] for b in range(self.B)]
