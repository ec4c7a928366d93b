"""Detection statistics on the GPU for max-pooling keyword models (SURVEY 8f-2).

Replaces the host round trip ``score.py`` (text score file, wekws/bin/score.py:128-137) ->
``compute_det.py`` (threshold sweep with ``window_shift`` skipping, wekws/bin/compute_det.py:76-105)
with one kernel over the posteriors that are already on the device, bit-exact with that pipeline.  The DET statistics
of CTC score files (``compute_det_ctc.py``) are per utterance and tiny; they run on the host (``ctc_det_stats``).
"""
from __future__ import annotations

import os
import re
from typing import Optional

import torch

from . import _native


def det_thresholds(step: float = 0.01) -> torch.Tensor:
    """The thresholds compute_det.py:79-105 visits: ``threshold = 0.0; while threshold <= 1.0: ...; threshold += step``
    accumulated in Python doubles."""
    out, threshold = [], 0.0
    while threshold <= 1.0:
        out.append(threshold)
        threshold += step
    return torch.tensor(out, dtype=torch.float64)


def det_stats(post: torch.Tensor, lengths: Optional[torch.Tensor] = None, step: float = 0.01,
              window_shift: int = 50):
    """post (B, T, K) float32 CUDA posteriors, lengths (B,) valid frames.  Returns (thresholds (n,) float64 on the
    host, max_score (B, K) float64, triggers (B, K, n) int32) -- see include/wekws_b200.h wekws_det_stats."""
    if not post.is_cuda:
        raise RuntimeError("wekws_b200.det_stats runs on CUDA only; got a CPU tensor (no CPU fallback)")
    if post.dim() != 3 or post.dtype != torch.float32:
        raise ValueError("post must be a (B, T, K) float32 tensor")
    post = post.contiguous()
    B, T, K = post.shape
    thr = det_thresholds(step)
    d_thr = thr.to(post.device)
    lens = None if lengths is None else lengths.to(device=post.device, dtype=torch.int32).contiguous()
    max_score = torch.empty(B, K, device=post.device, dtype=torch.float64)
    triggers = torch.empty(B, K, thr.numel(), device=post.device, dtype=torch.int32)
    _native.call("wekws_det_stats", post, lens, B, T, K, d_thr, thr.numel(), int(window_shift), max_score, triggers,
                 device=post.device)
    return thr, max_score, triggers


def det_curve(thresholds, max_score, triggers, is_keyword, filler_hours: float, keyword_index: int = 0):
    """Rows (threshold, false_alarm_per_hour, false_reject_rate) exactly as compute_det.py:98-104 writes them, from
    det_stats outputs: is_keyword (B,) bool marks the utterances whose transcript is the keyword."""
    is_keyword = torch.as_tensor(is_keyword, dtype=torch.bool).cpu()
    ms = max_score[:, keyword_index].double().cpu()
    tr = triggers[:, keyword_index].cpu()
    nk = int(is_keyword.sum())
    rows = []
    for i, th in enumerate(thresholds.tolist()):
        num_false_reject = int((ms[is_keyword] < th).sum())
        num_false_alarm = max(int(tr[~is_keyword, i].sum()), 1e-6)
        frr = num_false_reject / nk if nk else 0.0
        fa = num_false_alarm / filler_hours if filler_hours else 0.0
        rows.append((th, fa, frr))
    return rows


def split_mixed_label(input_str: str):
    """wekws/bin/compute_det_ctc.py:30-41: lower-cased Latin words (with !?,<>()' ) as one token, any other character
    on its own."""
    tokens = []
    s = input_str.lower()
    while len(s) > 0:
        match = re.match(r'[A-Za-z!?,<>()\']+', s)
        word = match.group(0) if match is not None else s[0:1]
        tokens.append(word)
        s = s.replace(word, '', 1).strip(' ')
    return tokens


def space_mixed_label(input_str: str) -> str:
    """compute_det_ctc.py:44-47: the tokens of split_mixed_label joined by single blanks."""
    return ''.join(f'{sub} ' for sub in split_mixed_label(input_str)).strip()


def ctc_det_stats(score_lines, labels, keywords, step: float = 0.01):
    """The DET statistics of wekws/bin/compute_det_ctc.py:50-124,228-281 for a CTC score file (score_ctc.py or
    stream_score_ctc.py; see write_ctc_scores / write_stream_ctc_scores).

    score_lines: the score file's lines (a str is the whole text); labels: (key, txt, duration) triples of the test set's
    data.list; keywords: {keyword as passed to --keywords: its token string} (the reference's ``true_keywords``).
    Returns {space_mixed_label(token string): [(threshold, false_alarm_per_hour, false_reject_rate), ...]} in keyword
    order, the rows of each stats.<keyword>.txt.  As the reference does: the first line of a key wins, a positive
    utterance detected as another keyword scores -1.0, a duplicate label key replaces its table entry but adds its
    duration again, and at least 1e-6 false alarms are counted."""
    if isinstance(score_lines, str):
        score_lines = score_lines.splitlines()
    score_table = {}
    for line in score_lines:
        arr = line.strip().split()
        if not arr:
            continue
        key = arr[0]
        if key in score_table:
            continue
        if arr[1] == 'detected':
            score_table[key] = {'kw': space_mixed_label(keywords[arr[2]]), 'confi': float(arr[3])}
        else:
            score_table[key] = {'kw': 'unknown', 'confi': -1.0}
    names = [space_mixed_label(keywords[k]) for k in keywords]
    table = {kw: {'keyword_table': {}, 'keyword_duration': 0.0, 'filler_table': {}, 'filler_duration': 0.0}
             for kw in names}
    for key, txt, duration in labels:
        if key not in score_table:
            raise ValueError(f"utterance {key!r} of the labels has no line in the score file")
        txt_lrblk = ' ' + space_mixed_label(txt) + ' '
        for kw in names:
            confi = score_table[key]['confi'] if kw == score_table[key]['kw'] else -1.0
            if txt_lrblk.find(' ' + kw + ' ') != -1:
                table[kw]['keyword_table'][key] = confi
                table[kw]['keyword_duration'] += duration
            else:
                table[kw]['filler_table'][key] = confi
                table[kw]['filler_duration'] += duration
    thresholds = det_thresholds(step).tolist()
    out = {}
    for kw in names:
        kw_conf = list(table[kw]['keyword_table'].values())
        filler_conf = list(table[kw]['filler_table'].values())
        if not kw_conf:
            raise ValueError(f"can't compute det for {kw} without positive sample")
        if not filler_conf:
            raise ValueError(f"can't compute det for {kw} without negative sample")
        filler_hours = table[kw]['filler_duration'] / 3600.0
        rows = []
        for threshold in thresholds:
            num_false_reject = sum(1 for c in kw_conf if c < threshold)
            num_false_alarm = max(sum(1 for c in filler_conf if c >= threshold), 1e-6)
            rows.append((threshold, num_false_alarm / filler_hours, num_false_reject / len(kw_conf)))
        out[kw] = rows
    return out


def write_ctc_det_stats(stats_dir: str, stats) -> list:
    """Writes each keyword's rows of ctc_det_stats to stats_dir/stats.<keyword with '_' for ' '>.txt exactly as
    compute_det_ctc.py:249-281 does ('{:.3f} {:.6f} {:.6f}').  Returns the paths written."""
    paths = []
    for kw, rows in stats.items():
        path = os.path.join(stats_dir, 'stats.' + kw.replace(' ', '_') + '.txt')
        with open(path, 'w', encoding='utf8') as fout:
            for row in rows:
                fout.write('{:.3f} {:.6f} {:.6f}\n'.format(*row))
        paths.append(path)
    return paths


def context_expansion(feats: torch.Tensor, left: int = 1, right: int = 1, skip_rate: int = 1,
                      lengths: Optional[torch.Tensor] = None):
    """wekws/dataset/processor.py:267-312 (context_expansion then frame_skip) on the device, batched:
    feats (B, T, D) float32 CUDA [, lengths (B,)] -> (expanded (B, m, D*(left+right+1)), new_lengths (B,) int32) with
    m = ceil((T - right) / skip_rate); stream b keeps ceil((lengths[b] - right) / skip_rate) rows, the rest are zero
    (the zero padding pad_sequence would add)."""
    if not feats.is_cuda:
        raise RuntimeError("wekws_b200.context_expansion runs on CUDA only; got a CPU tensor (no CPU fallback)")
    if feats.dim() != 3 or feats.dtype != torch.float32:
        raise ValueError("feats must be a (B, T, D) float32 tensor")
    feats = feats.contiguous()
    B, T, D = feats.shape
    m = int(_native.lib().wekws_context_expand_frames(T, int(right), int(skip_rate)))
    out = torch.empty(B, m, D * (left + right + 1), device=feats.device, dtype=torch.float32)
    lens = None if lengths is None else lengths.to(device=feats.device, dtype=torch.int32).contiguous()
    _native.call("wekws_context_expand", feats, lens, B, T, D, int(left), int(right), int(skip_rate), out, m,
                 device=feats.device)
    n = torch.full((B,), T, dtype=torch.int64) if lengths is None else lengths.detach().cpu().to(torch.int64)
    new_len = torch.where(n > right, (n - right + skip_rate - 1) // skip_rate, torch.zeros_like(n)).to(torch.int32)
    return out, new_len
