"""Held-out loss and accuracy on the device with the reference's training criteria.

``criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False)`` is a drop-in for
``wekws/model/loss.py`` ``criterion()`` with the same return contract: ``(loss, acc)``, ``loss`` a 0-dim float32
CUDA tensor and ``acc`` a Python float.  After ``wekws.utils.executor.criterion = wekws_b200.criterion`` the
reference's own ``Executor.cv`` / ``Executor.test`` evaluate a set with it.  The kernels are in csrc/criterion.cu:

* ``max_pooling`` (loss.py:26-88): the loss is the reference's float32 sum in (utterance, keyword) order;
* ``ce`` (loss.py:91-100,167-180): ``F.cross_entropy`` (mean, ``ignore_index=-100``) and ``acc_frame``;
* ``ctc`` (loss.py:102-164): ``F.ctc_loss(log_softmax, ..., blank=0, reduction='sum') / B`` (+inf for an infeasible
  utterance, as ``zero_infinity=False`` gives) and, with ``validation=True``, ``acc_utterance``: prefix beam search
  (score beam 3, path beam 5) on the softmax and the word accuracy of the best hypothesis against the label.

Training (``Executor.train``): when ``logits.requires_grad`` and grad mode is on, the returned loss is attached to
the graph, and ``loss.backward()`` delivers ``d loss / d logits`` -- the gradient torch's autograd gives for
``loss.py``, computed by the backward kernels of csrc/criterion.cu -- as a float32 tensor of the logits' shape.
Otherwise the forward-only entry points run, exactly as before.  Double backward is not supported.
"""
from __future__ import annotations

import math
import sys

import torch
from torch.autograd.function import once_differentiable

from . import _native
from ._native import CRITERION_MAX_LABEL as MAX_LABEL
from ._native import CTC_MAX_PREFIX as MAX_PREFIX      # longest hypothesis the accuracy decode keeps

IGNORE_INDEX = -100          # F.cross_entropy's default, part of the reference's contract
_INTS = (torch.int8, torch.int16, torch.int32, torch.int64, torch.uint8)


def criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    """wekws/model/loss.py criterion() on the device -> (loss: 0-dim float32 CUDA tensor, acc: float)."""
    if type == "ce":
        loss, acc, _ = cross_entropy(logits, target)
    elif type == "max_pooling":
        loss, acc, _ = max_pooling_loss(logits, target, lengths, min_duration)
    elif type == "ctc":
        loss, acc, _ = ctc_loss(logits, target, lengths, target_lengths, validation)
    else:
        sys.exit(1)
    return loss, acc


def _logits(x, dim):
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        raise ValueError("criterion: logits must be a CUDA tensor (there is no CPU path)")
    if x.dtype != torch.float32 or x.dim() != dim:
        raise ValueError(f"criterion: logits must be a {dim}-D float32 tensor, got {x.dim()}-D {x.dtype}")
    if x.shape[0] == 0:
        raise ValueError("criterion: empty batch")
    return x.contiguous()


def _ints(name, t, x, dim=1, size=None):
    if not isinstance(t, torch.Tensor) or t.device != x.device:
        raise ValueError(f"criterion: {name} must be a tensor on {x.device}")
    if t.dtype not in _INTS or t.dim() != dim or (size is not None and t.shape[0] != size):
        raise ValueError(f"criterion: {name} must be a {dim}-D integer tensor of {size} rows")
    return t


def _wants_grad(logits):
    return torch.is_grad_enabled() and logits.requires_grad


def _upstream(g, x):
    """The gradient arriving at the loss: the kernels read one float32 from device memory."""
    if g.dim() != 0 or g.dtype != torch.float32 or g.device != x.device:
        raise ValueError(f"criterion: the loss is a 0-dim float32 tensor on {x.device}; its upstream gradient must "
                         f"be one too, got {tuple(g.shape)} {g.dtype} on {g.device}")
    return g.contiguous()


class _MaxPoolingLoss(torch.autograd.Function):
    """The loss of wekws_criterion_max_pooling_train; ``args`` are the forward entry point's, from B to d_correct."""

    @staticmethod
    def forward(ctx, x, tgt, lens, *args):
        B, T, D, min_duration = args[:4]
        pooled = torch.empty(B, D, dtype=torch.float32, device=x.device)
        loss = torch.empty_like(args[5])
        _native.call("wekws_criterion_max_pooling_train", x, tgt, lens, *args[:5], loss, *args[6:], pooled,
                     device=x.device)
        ctx.save_for_backward(x, tgt, lens, pooled)
        ctx.min_duration = min_duration
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, tgt, lens, pooled = ctx.saved_tensors
        grad = torch.empty_like(x)
        _native.call("wekws_criterion_max_pooling_backward", x, tgt, lens, *x.shape, ctx.min_duration, pooled,
                     _upstream(g, x), grad, device=x.device)
        return (grad,) + (None,) * (len(ctx.needs_input_grad) - 1)


class _CrossEntropyLoss(torch.autograd.Function):
    """The loss of wekws_criterion_ce_train; ``args`` are the forward entry point's, from B to d_correct."""

    @staticmethod
    def forward(ctx, x, tgt, *args):
        count = torch.empty((), dtype=torch.float32, device=x.device)
        loss = torch.empty_like(args[3])
        _native.call("wekws_criterion_ce_train", x, tgt, *args[:3], loss, *args[4:], count, device=x.device)
        ctx.save_for_backward(x, tgt, count)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, tgt, count = ctx.saved_tensors
        grad = torch.empty_like(x)
        _native.call("wekws_criterion_ce_backward", x, tgt, *x.shape, count, _upstream(g, x), grad, device=x.device)
        return (grad,) + (None,) * (len(ctx.needs_input_grad) - 1)


class _CtcLoss(torch.autograd.Function):
    """The loss of wekws_criterion_ctc_train; ``args`` are the forward entry point's, from B to d_best.  Keeps alpha
    (B, T, 2 Lmax + 1), which the first backward turns into the state occupancies in place."""

    @staticmethod
    def forward(ctx, x, lens, *args):
        B, T, V, lab, stride, tls, max_label = args[:7]
        utt, loss = args[11], torch.empty_like(args[9])
        row_max = torch.empty(B, T, dtype=torch.float32, device=x.device)
        row_sum = torch.empty(B, T, dtype=torch.float32, device=x.device)
        alpha = torch.empty(B, T, 2 * max_label + 1, dtype=torch.float32, device=x.device)
        _native.call("wekws_criterion_ctc_train", x, lens, *args[:9], loss, *args[10:], row_max, row_sum, alpha,
                     device=x.device)
        ctx.save_for_backward(x, lens, lab, tls, row_max, row_sum, utt)
        ctx.alpha, ctx.stride, ctx.max_label, ctx.occupancy = alpha, stride, max_label, False
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        x, lens, lab, tls, row_max, row_sum, utt = ctx.saved_tensors
        grad = torch.empty_like(x)
        _native.call("wekws_criterion_ctc_backward", x, lens, *x.shape, lab, ctx.stride, tls, ctx.max_label, row_max,
                     row_sum, utt, ctx.alpha, int(ctx.occupancy), _upstream(g, x), grad, device=x.device)
        ctx.occupancy = True
        return (grad,) + (None,) * (len(ctx.needs_input_grad) - 1)


def max_pooling_loss(logits, target, lengths, min_duration=0, terms=False):
    """loss.py:26-88.  logits (B, T, D) posteriors, target (B,) (< 0 = filler), lengths (B,) with max == T.
    terms=True also returns {'term': (B, D) losses, 'correct': (B,) 0/1}."""
    x = _logits(logits, 3)
    B, T, D = x.shape
    target = _ints("target", target, x, size=B)
    lengths = _ints("lengths", lengths, x, size=B)
    if int(min_duration) < 0:
        raise ValueError("criterion: min_duration must be >= 0")
    lens_h = lengths.cpu()
    if int(lens_h.min()) < 0 or int(lens_h.max()) != T:
        raise ValueError(f"criterion: max_pooling needs logits of T = lengths.max() frames (T = {T}, lengths.max() = "
                         f"{int(lens_h.max())}): the reference's padding mask does not broadcast otherwise")
    tgt = target.clamp(-1, D).to(torch.int32)          # < 0: filler, D: no keyword column -- the reference's cases
    lens = lengths.to(torch.int32)
    ws = torch.empty(int(_native.lib().wekws_criterion_max_pooling_workspace_bytes(B, D)), dtype=torch.uint8,
                     device=x.device)
    loss = torch.empty((), dtype=torch.float32, device=x.device)
    acc = torch.empty(1, dtype=torch.float64, device=x.device)
    out = dict(term=torch.empty(B, D, dtype=torch.float32, device=x.device),
               correct=torch.empty(B, dtype=torch.int32, device=x.device)) if terms else {}
    args = (x, tgt, lens, B, T, D, int(min_duration), ws, loss, acc, out.get("term"), out.get("correct"))
    if _wants_grad(x):
        loss = _MaxPoolingLoss.apply(*args)
    else:
        _native.call("wekws_criterion_max_pooling", *args, device=x.device)
    return loss, float(acc.item()), out


def cross_entropy(logits, target, terms=False):
    """loss.py:167-180.  logits (B, C), target (B,) in 0..C-1 or -100 (ignored).
    terms=True also returns {'term': (B,) losses (unset where ignored), 'correct': (B,) 0/1}."""
    x = _logits(logits, 2)
    B, Cn = x.shape
    target = _ints("target", target, x, size=B)
    bad = (target != IGNORE_INDEX) & ((target < 0) | (target >= Cn))
    if bool(bad.any()):
        raise IndexError(f"Target {int(target[bad][0])} is out of bounds.")
    tgt = target.to(torch.int32)
    ws = torch.empty(int(_native.lib().wekws_criterion_ce_workspace_bytes(B)), dtype=torch.uint8, device=x.device)
    loss = torch.empty((), dtype=torch.float32, device=x.device)
    acc = torch.empty(1, dtype=torch.float64, device=x.device)
    out = dict(term=torch.empty(B, dtype=torch.float32, device=x.device),
               correct=torch.empty(B, dtype=torch.int32, device=x.device)) if terms else {}
    args = (x, tgt, B, Cn, ws, loss, acc, out.get("term"), out.get("correct"))
    if _wants_grad(x):
        loss = _CrossEntropyLoss.apply(*args)
    else:
        _native.call("wekws_criterion_ce", *args, device=x.device)
    return loss, float(acc.item()), out


def ctc_loss(logits, target, lengths, target_lengths, validation=False, terms=False):
    """loss.py:102-164.  logits (B, T, V), target (B, Lmax) padded (any padding value) or 1-D concatenated labels,
    lengths (B,) <= T, target_lengths (B,).  terms=True also returns {'term': (B,) per-utterance losses} and, with
    validation, 'correct': (B,) label length - edit distance, 'best': (B, 1 + 64) best hypothesis (length, tokens)."""
    x = _logits(logits, 3)
    B, T, V = x.shape
    lengths = _ints("lengths", lengths, x, size=B)
    target_lengths = _ints("target_lengths", target_lengths, x, size=B)
    if not isinstance(target, torch.Tensor) or target.dim() not in (1, 2):
        raise ValueError("criterion: ctc target must be a (B, Lmax) or 1-D integer tensor")
    target = _ints("target", target, x, dim=target.dim())
    if target.dim() == 1 and validation:
        # acc_utterance indexes target[i][:len]: the 1-D target Executor.cv makes when Lmax == 1 cannot be indexed so
        raise IndexError("criterion: validation needs (B, Lmax) targets; target[i] of a 1-D target is a 0-dim tensor")
    if target.dim() == 2 and target.shape[0] != B:
        raise ValueError("criterion: target must have B rows")
    n_lab = target.shape[1] if target.dim() == 2 else target.numel()
    tl = target_lengths.to(torch.int64)
    pos = torch.arange(n_lab, device=x.device)
    valid = pos[None, :] < tl[:, None] if target.dim() == 2 else pos < tl.sum()
    bad = (((target < 0) | (target >= V)) & valid).any()
    host = torch.cat([lengths.to(torch.int64), tl, bad.view(1).to(torch.int64)]).cpu()
    lens_h, tl_h = host[:B], host[B:2 * B]
    if int(lens_h.min()) < 0 or int(lens_h.max()) > T:
        raise ValueError(f"criterion: lengths must be in 0..{T}")
    if int(tl_h.min()) < 0 or (int(tl_h.max()) > n_lab if target.dim() == 2 else int(tl_h.sum()) > n_lab):
        raise ValueError("criterion: target_lengths exceed the target tensor")
    if int(tl_h.max()) > MAX_LABEL:
        raise ValueError(f"criterion: ctc labels of up to {MAX_LABEL} tokens are supported, got {int(tl_h.max())}")
    if int(host[-1]):
        raise ValueError(f"criterion: ctc labels must be token ids in 0..{V - 1}")
    if validation and V < 3:
        raise ValueError("criterion: the accuracy decode takes the top 3 tokens per frame; V must be >= 3")
    lab = target.to(torch.int32).contiguous()
    lens = lengths.to(torch.int32)
    tls = target_lengths.to(torch.int32)
    dev = x.device
    ws = torch.empty(int(_native.lib().wekws_criterion_ctc_workspace_bytes(B, T, int(bool(validation)))),
                     dtype=torch.uint8, device=dev)
    loss = torch.empty((), dtype=torch.float32, device=dev)
    acc = torch.empty(1, dtype=torch.float64, device=dev)
    overflow = torch.empty(B, dtype=torch.int32, device=dev) if validation else None
    out = {}
    if terms:
        out["term"] = torch.empty(B, dtype=torch.float32, device=dev)
        if validation:
            out["correct"] = torch.empty(B, dtype=torch.int32, device=dev)
            out["best"] = torch.empty(B, 1 + MAX_PREFIX, dtype=torch.int32, device=dev)
    stride = n_lab if target.dim() == 2 else 0
    args = (x, lens, B, T, V, lab, stride, tls, int(tl_h.max()), int(bool(validation)), ws, loss, acc,
            out.get("term"), out.get("correct"), overflow, out.get("best"))
    if _wants_grad(x):                                    # the backward needs the per-utterance losses
        utt = out["term"] if terms else torch.empty(B, dtype=torch.float32, device=dev)
        loss = _CtcLoss.apply(*args[:13], utt, *args[14:])
    else:
        _native.call("wekws_criterion_ctc", *args, device=dev)
    if not validation:
        return loss, 0.0, out
    res = torch.cat([acc, overflow.to(torch.float64)]).cpu()
    over = res[1:].nonzero().flatten().tolist()
    if over:
        raise RuntimeError(f"criterion: the CTC decode of utterance {over[0]} outgrew {MAX_PREFIX} tokens, so its "
                           "accuracy would not be the reference's")
    a = float(res[0])
    if math.isnan(a):
        raise ZeroDivisionError("float division by zero (every label of the batch is empty)")
    return loss, a, out
