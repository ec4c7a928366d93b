"""Gradients of the reference's training criteria and its training loop, for tests only: the companion of
kws_criterion_oracle.py (the forward restatement of wekws/model/loss.py criterion()).

* `criterion_grad` differentiates the criteria with torch's autograd in float32 or float64: max_pooling through
  `max_pooling_loss_graph`, which pools each (utterance, keyword) column with the full max() / min() reductions the
  reference uses, so ties split as they do there; ce and ctc through the forward restatement.
* `ctc_grad_closed_form` is the formula the device kernels implement, (softmax - occupancy) / B, from its own alpha /
  beta recurrence.
* `train` restates wekws/utils/executor.py Executor.train's loop.
The golden tests/golden/criterion_grad.npz pins `criterion_grad` against the reference's own loss.py.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .kws_criterion_oracle import ctc_loss


def max_pooling_loss_graph(logits, target, lengths, min_duration=0):
    """The loss of loss.py:46-71 as a graph: per (utterance, keyword) column the masked, clamped posteriors reduced by
    a full max() / min(), whose backward splits the gradient evenly over the tied positions."""
    B, T, D = logits.shape
    mask = torch.arange(T)[None, :] >= lengths.long()[:, None]
    loss = 0.0
    for i in range(B):
        for j in range(D):
            if int(target[i]) == j:
                m = mask[i].clone()
                m[:min_duration] = True
                pooled = logits[i, :, j].masked_fill(m, 0.0).clamp(1e-8, 1.0).max()
            else:
                pooled = (1 - logits[i, :, j]).masked_fill(mask[i], 1.0).clamp(1e-8, 1.0).min()
            loss = loss + -torch.log(pooled)
    return loss / B


def criterion_grad(type, logits, target, lengths, target_lengths=None, min_duration=0, upstream=1.0,
                   dtype=torch.float32):
    """(loss, d (upstream * loss) / d logits) in `dtype` by autograd; the gradient has the logits' shape."""
    x = logits.detach().to(dtype).clone().requires_grad_(True)
    if type == "max_pooling":
        loss = max_pooling_loss_graph(x, target, lengths, min_duration)
    elif type == "ce":
        loss = F.cross_entropy(x, target.long())
    elif type == "ctc":
        loss = ctc_loss(x, target, lengths, target_lengths)[0]
    else:
        raise SystemExit(1)
    (loss * upstream).backward()
    return loss.detach(), x.grad


def ctc_grad_closed_form(logits, target, lengths, target_lengths):
    """d ctc_loss / d logits in float64 without autograd: (softmax - occupancy) / B on the frames of a feasible
    utterance, where the occupancy of token v at frame t is the sum over the extended-label states s carrying v of
    exp(alpha[t, s] + beta[t, s] - log p(label)); zero on padding frames.  target is (B, Lmax).  Also returns the
    per-frame total occupancy (B, T), which is 1 on every frame of a feasible utterance."""
    x = logits.double()
    B, T, V = x.shape
    lp = x.log_softmax(2)
    grad = torch.zeros_like(x)
    total = torch.zeros(B, T, dtype=torch.float64)
    ninf = float("-inf")
    for b in range(B):
        n, L = int(lengths[b]), int(target_lengths[b])
        ext = [0] * (2 * L + 1)
        ext[1::2] = [int(v) for v in target[b][:L]]
        S = len(ext)
        if n == 0:
            continue
        e = lp[b][:, ext]                                 # (T, S) log-probability of each state's token
        alpha = torch.full((n, S), ninf, dtype=torch.float64)
        beta = torch.full((n, S), ninf, dtype=torch.float64)
        alpha[0, :2] = e[0, :2]
        beta[n - 1, S - 2:] = e[n - 1, S - 2:]
        lse = lambda vals: torch.logsumexp(torch.stack(vals), 0) if max(vals) > ninf else torch.tensor(ninf).double()
        for t in range(1, n):
            for s in range(S):
                prev = [alpha[t - 1, s]] + ([alpha[t - 1, s - 1]] if s > 0 else [])
                if s > 1 and ext[s] != 0 and ext[s] != ext[s - 2]:
                    prev.append(alpha[t - 1, s - 2])
                alpha[t, s] = lse(prev) + e[t, s]
        for t in range(n - 2, -1, -1):
            for s in range(S):
                nxt = [beta[t + 1, s]] + ([beta[t + 1, s + 1]] if s + 1 < S else [])
                if s + 2 < S and ext[s] != 0 and ext[s] != ext[s + 2]:
                    nxt.append(beta[t + 1, s + 2])
                beta[t, s] = lse(nxt) + e[t, s]
        log_p = torch.logsumexp(alpha[n - 1, S - 2:], 0)
        gamma = (alpha + beta - e[:n] - log_p).exp()      # (n, S)
        total[b, :n] = gamma.sum(1)
        occ = torch.zeros(n, V, dtype=torch.float64).index_add_(1, torch.tensor(ext), gamma)
        grad[b, :n] = (lp[b, :n].exp() - occ) / B
    return grad, total


def train(crit, model, optimizer, batches, device, args):
    """Executor.train (executor.py:28-68) with `crit` in place of the criterion it imports: one optimiser step per
    batch after clip_grad_norm_, skipped when the gradient norm is not finite.  Returns [(loss, stepped)]."""
    model.train()
    clip = args.get("grad_clip", 50.0)
    min_duration = args.get("min_duration", 0)
    log = []
    for batch in batches:
        target = batch["target"]
        target = target[:, 0] if target.shape[1] == 1 else target
        feats_lengths = batch["feats_lengths"].to(device)
        if feats_lengths.size(0) == 0:
            continue
        logits, _ = model(batch["feats"].to(device))
        loss, acc = crit(args.get("criterion", "max_pooling"), logits, target.to(device), feats_lengths,
                         target_lengths=batch["target_lengths"].to(device), min_duration=min_duration,
                         validation=False)
        optimizer.zero_grad()
        loss.backward()
        grad_norm = torch.nn.utils.clip_grad_norm_(model.parameters(), clip)
        stepped = bool(torch.isfinite(grad_norm))
        if stepped:
            optimizer.step()
        log.append((loss.item(), stepped))
    return log
