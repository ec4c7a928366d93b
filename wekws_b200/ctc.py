"""CTC prefix beam search and keyword look-up on the GPU (SURVEY 8f-2, CTC models).

Replaces the per-utterance / per-frame pure-Python decoding of the reference -- ``wekws/model/loss.py:206-312``
(``ctc_prefix_beam_search``) as called by ``wekws/bin/score_ctc.py:198-226`` and its streaming twin
``wekws/bin/stream_kws_ctc.py:124-215,400-434`` -- with one kernel over all utterances, bit-exact (hypothesis
order, scores as doubles, node frames / probabilities; see csrc/ctc_decode.cu for the Python semantics it keeps).
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Iterable, List, Optional, Sequence

import torch

from . import _native

MAX_PREFIX, MAX_PATH_BEAM, MAX_SCORE_BEAM = 64, 20, 3


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

    def p(t):
        return C.c_void_p(t.data_ptr()) if t is not None else None

    with torch.cuda.device(dev):
        rc = _native.lib().wekws_ctc_prefix_beam_search(
            p(probs), p(lens), B, T, V, p(kw), 0 if kw is None else kw.numel(), int(score_beam_size), int(path_beam_size),
            int(frame_offset), int(frame_stride), p(state), 1 if reset_state else 0, p(out.nhyp), p(out.hyp_len),
            p(out.hyp_tokens), p(out.hyp_score), p(out.node_frame), p(out.node_prob), p(out.overflow),
            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    _native.check(rc, "wekws_ctc_prefix_beam_search")
    return out


def ctc_keyword_hits(hyps: CtcHyps, keywords_token: Dict[str, dict]):
    """score_ctc.py:201-220 on the device: for every utterance the first hypothesis (beam order) that contains a keyword
    (dict order) -> list of (word or None, hit_score, start_frame, end_frame).  keywords_token: {word: {'token_id':
    [...]}} as the reference builds it (score_ctc.py:159-171)."""
    words = list(keywords_token.keys())
    seqs = [list(keywords_token[w]["token_id"]) for w in words]
    dev = hyps.nhyp.device
    flat = torch.tensor([t for s in seqs for t in s], dtype=torch.int32, device=dev)
    offs = [0]
    for s in seqs:
        offs.append(offs[-1] + len(s))
    offs = torch.tensor(offs, dtype=torch.int32, device=dev)
    hit = torch.empty(hyps.B, dtype=torch.int32, device=dev)
    score = torch.empty(hyps.B, dtype=torch.float64, device=dev)
    start = torch.empty(hyps.B, dtype=torch.int32, device=dev)
    end = torch.empty(hyps.B, dtype=torch.int32, device=dev)

    def p(t):
        return C.c_void_p(t.data_ptr())

    with torch.cuda.device(dev):
        rc = _native.lib().wekws_ctc_keyword_hit(
            p(hyps.nhyp), p(hyps.hyp_len), p(hyps.hyp_tokens), p(hyps.node_frame), p(hyps.node_prob), hyps.B,
            hyps.path_beam, p(flat), p(offs), len(words), p(hit), p(score), p(start), p(end),
            C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    _native.check(rc, "wekws_ctc_keyword_hit")
    hit, score, start, end = hit.cpu().tolist(), score.cpu().tolist(), start.cpu().tolist(), end.cpu().tolist()
    return [(words[h] if h >= 0 else None, score[b], start[b], end[b]) for b, h in enumerate(hit)]


def write_ctc_scores(fout, keys: Sequence[str], hits) -> None:
    """The score file of score_ctc.py:217-226: '{key} detected {keyword} {score:.3f}' or '{key} rejected'."""
    for key, (word, hit_score, _, _) in zip(keys, hits):
        if word is not None:
            fout.write('{} detected {} {:.3f}\n'.format(key, word, hit_score))
        else:
            fout.write('{} rejected\n'.format(key))


# one wekws_ctc_spot_result per stream (include/wekws_b200.h)
SPOT_RESULT_DTYPE = [("score", "<f8"), ("state", "<i4"), ("keyword", "<i4"), ("start", "<i4"), ("end", "<i4"),
                     ("overflow", "<i4"), ("reserved", "<i4")]
SPOT_RESULT_BYTES = 32


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
        offs = [0]
        for s in seqs:
            offs.append(offs[-1] + len(s))
        self._set = torch.tensor(sorted(tokenset), dtype=torch.int32, device=self.dev)
        self._kw = torch.tensor([t for s in seqs for t in s], dtype=torch.int32, device=self.dev)
        self._off = torch.tensor(offs, dtype=torch.int32, device=self.dev)
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

        def p(t):
            return C.c_void_p(t.data_ptr())

        with torch.cuda.device(self.dev):
            rc = _native.lib().wekws_ctc_spot(
                p(probs), V, p(rows), p(frames), self.B, p(self._set), self._set.numel(), p(self._kw), p(self._off),
                len(self.words), self.score_beam, self.path_beam, self.frame_stride, self.threshold, self.min_frames,
                self.max_frames, self.interval_frames, p(self.state), p(self.det), p(self.result),
                C.c_void_p(torch.cuda.current_stream(self.dev).cuda_stream))
        _native.check(rc, "wekws_ctc_spot")
        return self.result

    def hypotheses(self) -> List[list]:
        """Each stream's carried hypotheses as [(prefix, pb + pnb, nodes)] (hyps_of(cur_hyps))."""
        out = ctc_prefix_beam_search(torch.empty(self.B, 0, 1, device=self.dev), None, None, 1, self.path_beam,
                                     state=self.state, reset_state=False).to_python()
        return [out[b] if self._live[b] else [(tuple(), 1.0, [])] for b in range(self.B)]
