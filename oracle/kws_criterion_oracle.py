"""CPU restatement of the reference's training criteria (wekws/model/loss.py criterion(): max_pooling, ce, ctc) and of
the aggregation of wekws/utils/executor.py Executor.cv, for tests only.

* max_pooling: per-term values with the reference's own torch ops on the same 0-dim tensors (so the same log
  path), folded in float32 in (utterance, keyword) order, / B.
* ce: F.cross_entropy and acc_frame as the reference writes them.
* ctc: F.ctc_loss on the log-softmax (reduction 'sum' / B, and 'none' for the per-utterance values); the accuracy
  decodes with the existing beam-search restatement (kws_oracle.ctc_prefix_beam_search, score beam 3, path beam 5)
  and takes the plain Levenshtein distance instead of Calculator's back-trace: that trace only steps to a
  predecessor whose distance differs by the step's cost, and `cor` costs 0, so ins + sub + del along it is the edit
  distance and `all` is the label length.  The golden (tests/golden/criterion.npz) pins this against Calculator.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import kws_oracle as O


def max_pooling_terms(logits, target, lengths, min_duration=0):
    """(B, D) float32 loss terms and the (B,) correct flags of loss.py:44-85."""
    B, T, D = logits.shape
    mask = torch.arange(T)[None, :] >= lengths.long()[:, None]
    kw_mask = mask.clone()
    kw_mask[:, :min_duration] = True
    kw = logits.masked_fill(kw_mask[:, :, None], 0.0).clamp(1e-8, 1.0).amax(1)        # (B, D)
    other = (1 - logits).masked_fill(mask[:, :, None], 1.0).clamp(1e-8, 1.0).amin(1)
    terms = torch.empty(B, D)
    for i in range(B):
        for j in range(D):
            terms[i, j] = -torch.log(kw[i, j] if int(target[i]) == j else other[i, j])
    max_logits = logits.masked_fill(mask[:, :, None], 0.0).max(1)[0]
    max_p, idx = max_logits.max(1)
    correct = [(bool(max_p[i] > 0.5) and int(idx[i]) == int(target[i])) or (bool(max_p[i] < 0.5) and int(target[i]) < 0)
               for i in range(B)]
    return terms, torch.tensor(correct, dtype=torch.int32)


def max_pooling_loss(logits, target, lengths, min_duration=0):
    terms, correct = max_pooling_terms(logits, target, lengths, min_duration)
    loss = torch.zeros((), dtype=torch.float32)
    for v in terms.flatten():
        loss = loss + v
    return loss / logits.size(0), int(correct.sum()) / logits.size(0)


def cross_entropy(logits, target):
    loss = F.cross_entropy(logits, target.long())
    pred = logits.max(1)[1]
    return loss, int((pred == target.long()).sum()) * 100.0 / logits.size(0)


def edit_distance(lab, rec):
    """Levenshtein distance with unit costs (Calculator's cost table)."""
    prev = list(range(len(rec) + 1))
    for i, a in enumerate(lab, 1):
        cur = [i]
        for j, r in enumerate(rec, 1):
            cur.append(min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (a != r)))
        prev = cur
    return prev[-1]


def best_hypotheses(logits, lengths):
    """acc_utterance's decode: the best prefix of ctc_prefix_beam_search(softmax[:len], len, None, 3, 5) per utterance."""
    probs = logits.softmax(2)
    out = []
    for b in range(logits.size(0)):
        hyps = O.hyps_of(O.ctc_prefix_beam_search(probs[b][:int(lengths[b])], None, 3, 5))
        out.append(tuple(hyps[0][0]) if hyps else ())
    return out


def ctc_utterance_losses(logits, target, lengths, target_lengths):
    lp = logits.transpose(0, 1).log_softmax(2)
    return F.ctc_loss(lp, target, lengths, target_lengths, reduction="none")


def ctc_counts(logits, target, lengths, target_lengths):
    """[(label length, label length - edit distance of the best hypothesis)] per utterance."""
    out = []
    for b, rec in enumerate(best_hypotheses(logits, lengths)):
        lab = target[b][:int(target_lengths[b])].tolist()
        out.append((len(lab), len(lab) - edit_distance(lab, list(rec))))
    return out


def ctc_loss(logits, target, lengths, target_lengths, validation=False):
    acc = 0.0
    if validation:
        counts = ctc_counts(logits, target, lengths, target_lengths)
        words = sum(n for n, _ in counts if n > 0)
        acc = float(sum(c for n, c in counts if n > 0)) * 100.0 / words
    lp = logits.transpose(0, 1).log_softmax(2)
    loss = F.ctc_loss(lp, target, lengths, target_lengths, reduction="sum")
    return loss / lp.size(1), acc


def criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    if type == "ce":
        return cross_entropy(logits, target)
    if type == "max_pooling":
        return max_pooling_loss(logits, target, lengths, min_duration)
    if type == "ctc":
        return ctc_loss(logits, target, lengths, target_lengths, validation)
    raise SystemExit(1)


def cv(crit, model, batches, device, args):
    """Executor.cv (executor.py:68-110) with `crit` in place of the criterion it imports: num_seen_utts starts at 1,
    batches with a non-finite loss are skipped, and the totals are doubles of loss.item() * num_utts."""
    num_seen_utts = 1
    total_loss = 0.0
    total_acc = 0.0
    with torch.no_grad():
        for batch in batches:
            target = batch["target"]
            target = target[:, 0] if target.shape[1] == 1 else target
            feats_lengths = batch["feats_lengths"].to(device)
            num_utts = feats_lengths.size(0)
            if num_utts == 0:
                continue
            logits, _ = model(batch["feats"].to(device))
            loss, acc = crit(args.get("criterion", "max_pooling"), logits, target.to(device), feats_lengths,
                             target_lengths=batch["target_lengths"].to(device), min_duration=0, validation=True)
            if torch.isfinite(loss):
                num_seen_utts += num_utts
                total_loss += loss.item() * num_utts
                total_acc += acc * num_utts
    return total_loss / num_seen_utts, total_acc / num_seen_utts
