"""CPU restatement of the reference's streaming scorer, one utterance (wekws/bin/stream_score_ctc.py:221-377), built
from the beam step of kws_oracle (``ctc_prefix_beam_search`` with carried hypotheses) and ``is_sublist``.  It states
the semantics wekws_b200.stream_score_ctc keeps:

* a frame whose filtered top-k is empty is skipped entirely: no hypothesis update and no detection;
* hit keyword, start, end and hit_score persist across frames and are reset only on activation (with the hypotheses),
  so once a keyword has been seen only the first hypothesis is searched and hit_score is square-rooted again on every
  later decoded frame;
* an activation does not end the utterance; there is no interval rule and no max_frames reset;
* frame numbers are t * frame_skip.

Pinned by tests/golden/stream_score.npz, made by running the reference's own main() (oracle/make_stream_score_golden.py).
"""
from __future__ import annotations

import math

from . import kws_oracle as O

ACTIVATED, LOW_SCORE, BAD_DURATION = 0, 1, 2


def _decoded(p, tokenset, score_beam):
    """stream_score_ctc.py:244-261: False if no top-k token passes the filter (the frame is skipped)."""
    probs, index = p.topk(score_beam)
    return any(prob > 0.05 and idx in tokenset for prob, idx in zip(probs.tolist(), index.tolist()))


def stream_score(probs, keywords, score_beam_size=3, path_beam_size=20, threshold=0.0, min_frames=5, max_frames=250,
                 frame_skip=1):
    """probs (n, V) float32 softmax rows of one utterance (its first lengths[b] rows); keywords {word: token ids} in
    --keywords order.  Returns (detections, events): detections [(word, score, start, end, frame)] in firing order;
    events [(kind, word, score, start, end, frame)], one per decoded frame that holds a (possibly stale) hit, kind
    ACTIVATED / LOW_SCORE / BAD_DURATION -- the log lines of :349-374."""
    kws = {w: tuple(int(t) for t in s) for w, s in keywords.items()}
    tokenset = {0}.union(*[set(s) for s in kws.values()])
    cur_hyps = [(tuple(), (1.0, 0.0, []))]
    hit_keyword, hit_score, start, end = None, 1.0, 0, 0
    detections, events = [], []
    for t in range(probs.shape[0]):
        if not _decoded(probs[t], tokenset, score_beam_size):
            continue
        frame = t * frame_skip
        cur_hyps = O.ctc_prefix_beam_search(probs[t:t + 1], tokenset, score_beam_size, path_beam_size,
                                            cur_hyps=cur_hyps, frame_offset=frame)
        for prefix, _, nodes in O.hyps_of(cur_hyps):
            for w, lab in kws.items():
                off = O.is_sublist(prefix, lab)
                if off != -1:
                    hit_keyword, start, end = w, nodes[off]['frame'], nodes[off + len(lab) - 1]['frame']
                    for i in range(off, off + len(lab)):
                        hit_score *= nodes[i]['prob']
                    break
            if hit_keyword is not None:
                hit_score = math.sqrt(hit_score)
                break
        if hit_keyword is None:
            continue
        duration = end - start
        if hit_score >= threshold and min_frames <= duration <= max_frames:
            detections.append((hit_keyword, hit_score, start, end, frame))
            events.append((ACTIVATED, hit_keyword, hit_score, start, end, frame))
            cur_hyps = [(tuple(), (1.0, 0.0, []))]
            hit_keyword, hit_score = None, 1.0
        elif hit_score < threshold:
            events.append((LOW_SCORE, hit_keyword, hit_score, start, end, frame))
        else:
            events.append((BAD_DURATION, hit_keyword, hit_score, start, end, frame))
    return detections, events


def score_lines(key, detections):
    """The score-file lines of :349-376 for one utterance."""
    if not detections:
        return ['{} rejected\n'.format(key)]
    return ['{} detected {} {:.3f}\n'.format(key, word, score) for word, score, _, _, _ in detections]
