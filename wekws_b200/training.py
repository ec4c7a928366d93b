"""Training on the device: the training-mode forward of a ``KWSModel`` and its backward, for ``Executor.train``.

Which models train, and how they opt in:

* FSMN: no opt-in.  In ``train()`` mode, with grad mode on and a parameter requiring grad, the logits are attached to
  the autograd graph and ``loss.backward()`` fills ``.grad`` of every parameter of the reference's FSMN
  (wekws/model/fsmn.py).  Under ``no_grad`` the call takes the eval path: the FSMN has no BatchNorm and its Dropout is
  never called, so the training-mode forward is the eval forward.  The forward is the fused kernel of csrc/fsmn.cu in
  its storing instantiation (its logits are the eval logits, bit for bit), the backward the kernels of
  csrc/fsmn_grad.cu.  Each forward first packs the parameters' current values into the model's native handle on the
  device (one launch), so ``optimizer.step()`` needs no host round trip; when the handle was rebuilt between the
  forward and the backward, the backward packs the same values again.
* GRU, after ``model.enable_training(bptt=True)``: as FSMN, with grad mode on and a parameter requiring grad the
  logits are attached to the autograd graph and ``loss.backward()`` fills ``.grad`` of every parameter (the
  preprocessing Linear, every layer of ``nn.GRU``, the classifier); without grad the call takes the eval path (the GRU
  model has no BatchNorm and no Dropout).  The forward is the FP32 kernel of csrc/gru.cu in its storing instantiation,
  whatever ``model.precision`` is (its logits and cache are the FP32 eval kernel's, bit for bit); the backward through
  time is csrc/gru_train.cu.  Parameters are packed into the handle on the device as for FSMN.  The opt-in is the
  caller's acceptance of the memory the forward keeps: (1 + 5 L) B T 128 floats.
* MDTC, after ``model.enable_training()``, and TCN / DS-TCN, after ``model.enable_training(device_dropout=True)``, each
  with the per-frame linear classifier: the training-mode forward of the reference's wekws/model/kws_model.py, with or
  without grad.  Every BatchNorm normalises with the biased variance of the batch (all B * T frames, padding included),
  updates ``running_mean`` / ``running_var`` (the latter with the unbiased variance) with its own ``momentum`` and
  ``eps``, and counts ``num_batches_tracked``.  With grad the logits are attached to the autograd graph; without, the
  same forward runs without keeping activations.  The kernels (csrc/mdtc_train.cu, csrc/tcn_train.cu) read the
  parameters, the CMVN buffers and the running statistics where they live on the device.  The running statistics are
  written by a kernel, behind the version counters' back, so each training forward marks the packed eval model stale:
  the next eval call repacks.  The opt-in exists because a BatchNorm model in training mode gives other outputs than in
  eval mode and overwrites its running statistics: a model left in ``train()`` by accident keeps refusing to run.

* MDTC with the ``global`` / ``last`` head (the speech-command recipe), after
  ``model.enable_training(device_dropout=True)``: the same backbone forward, then the head's training forward
  (Linear, ReLU, Dropout, Linear on the mean over the frames or on the last frame), logits (B, odim); the backward
  runs the head's kernels (csrc/mdtc_head_train.cu) and then the backbone's from the stack sum's gradient.

Dropout (TCN / DS-TCN blocks, the MDTC heads): no device generator reproduces torch's Bernoulli stream, so every
``nn.Dropout`` applies a mask that is a documented pure function of a 64-bit seed (include/wekws_b200.h,
``wekws_train_forward``).  The seed is one draw from torch's default CPU generator per training forward
(``frontend.draw_seed``), so ``torch.manual_seed`` makes a run reproducible; when every ``p`` is 0 nothing is drawn.
``p`` is read from the model's own ``nn.Dropout`` modules at call time.  The backward recomputes the masks from the
seed; they are never stored.  ``device_dropout=True`` is the caller's acceptance of these masks in place of torch's.

Refused: GRU training without ``bptt=True``, a GRU with inter-layer Dropout or outside the kernels' limits, and the
heads behind TCN / DS-TCN (at ``enable_training``); per call, ``forward_softmax``, a non-empty streaming cache,
features that require grad, ``momentum=None``, non-contiguous or non-float32 parameters, and double backward.  The
per-model names, orders, formulas and limits are in mdtc_train.py, tcn_train.py, fsmn_train.py and gru_train.py.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Tuple

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _native, fsmn_train, gru_train, mdtc_train, tcn_train


def _kind(model) -> Optional[str]:
    bb = model.backbone
    return "gru" if isinstance(bb, nn.GRU) else getattr(bb, "kind", None)


def _label(kind: str) -> str:
    return str(kind).upper().replace("_", "-")           # MDTC, TCN, DS-TCN, FSMN, GRU


def _batch_norms(model) -> List[nn.BatchNorm1d]:
    return (mdtc_train if model.backbone.kind == "mdtc" else tcn_train).batch_norms(model)


def check_trainable(model, device_dropout: bool, bptt: bool = False) -> None:
    """Raises NotImplementedError unless ``model.enable_training(device_dropout, bptt)`` can train `model`."""
    kind = _kind(model)
    if kind == "fsmn":
        return
    label = _label(kind)
    if kind == "gru":
        if not bptt:
            raise NotImplementedError("wekws_b200: training the GRU backbone keeps every step's gates for the backward "
                                      "through time, (1 + 5 num_layers) * B * T * 128 floats: opt in with "
                                      "model.enable_training(bptt=True)")
        gru_train.check_limits(model)
        return
    if kind in ("tcn", "ds_tcn") and not device_dropout:
        raise NotImplementedError(f"wekws_b200: training the {label} backbone applies Dropout masks made on the device, "
                                  "not torch's Bernoulli draws: opt in with model.enable_training(device_dropout=True)")
    if kind not in ("mdtc", "tcn", "ds_tcn"):
        raise NotImplementedError(f"wekws_b200: training is not implemented for the {label} backbone")
    if model.head is not None:
        if kind != "mdtc":
            raise NotImplementedError(f"wekws_b200: {label} training runs with the per-frame linear classifier; the "
                                      f"'{model.head}' head has Dropout and trains behind the MDTC backbone only")
        if not device_dropout:
            raise NotImplementedError(f"wekws_b200: the '{model.head}' head has Dropout, whose masks are made on the "
                                      "device, not torch's Bernoulli draws: opt in with "
                                      "model.enable_training(device_dropout=True)")
        if not isinstance(model.activation, nn.Identity):
            raise NotImplementedError(f"wekws_b200: MDTC training with the '{model.head}' head needs the Identity "
                                      "activation")
    if not isinstance(model.activation, (nn.Sigmoid, nn.Identity)):
        raise NotImplementedError(f"wekws_b200: {label} training needs the Sigmoid or Identity activation")
    (mdtc_train if kind == "mdtc" else tcn_train).check_limits(model)


def wants_grad(model) -> bool:
    """True when a training-mode call must build the autograd graph: grad mode on, a parameter requiring grad."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters())


def _check_inputs(x: torch.Tensor, in_cache: torch.Tensor, label: str, cache_refusal: str) -> None:
    if in_cache is not None and in_cache.numel() > 0:
        raise ValueError(f"wekws_b200: {label} training runs from empty caches (as Executor.train does); a streaming "
                         f"cache {cache_refusal}")
    if x.requires_grad:
        raise ValueError(f"wekws_b200: {label} training computes parameter gradients only; features that require grad "
                         "are not supported (detach them)")


def route(model, x: torch.Tensor, in_cache: torch.Tensor, flags: int) -> bool:
    """Whether a call of `model` in training mode runs ``forward`` (True) or the eval path (False, FSMN without grad).
    Raises the refusals that need no device."""
    kind = _kind(model)
    if kind == "gru" and not (model.__dict__.get("_training_enabled", False) and model.__dict__.get("_bptt", False)):
        raise RuntimeError("wekws_b200.KWSModel is inference-only: call model.eval() first "
                           "(training-mode BatchNorm/Dropout are not implemented) -- or call "
                           "model.enable_training(bptt=True) to train this GRU model")
    if kind in ("fsmn", "gru"):
        train = wants_grad(model)
    else:
        enabled = model.__dict__.get("_training_enabled", False)
        dropout = kind in ("tcn", "ds_tcn") or kind == "mdtc" and model.head is not None
        if not (enabled and kind in ("mdtc", "tcn", "ds_tcn") and (not dropout or model.__dict__.get("_device_dropout"))):
            hint = (" -- or call model.enable_training(device_dropout=True) to train this model" if dropout else
                    " -- or call model.enable_training() to train this MDTC model" if kind == "mdtc" else "")
            raise RuntimeError("wekws_b200.KWSModel is inference-only: call model.eval() first "
                               "(training-mode BatchNorm/Dropout are not implemented)" + hint)
        train = True
    if train and flags != 0:
        raise RuntimeError("wekws_b200: forward_softmax has no training path; call forward() for training")
    if kind not in ("fsmn", "gru"):
        label = _label(kind)
        _check_inputs(x, in_cache, label, "is not supported in training mode -- pass no in_cache, or call model.eval()")
        if x.dim() == 3 and x.shape[0] * x.shape[1] <= 1:
            raise ValueError("Expected more than 1 value per channel when training, got input size "
                             f"{torch.Size([x.shape[0], model.hdim, x.shape[1]])}")
        for bn in _batch_norms(model):
            if bn.momentum is None:
                raise ValueError("wekws_b200: BatchNorm momentum=None (a cumulative moving average) is not supported "
                                 f"in {label} training; set a momentum")
    return train


def _pointers(tensors) -> C.Array:
    return (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _params(model, dev: torch.device, names: List[str], label: str) -> List[torch.Tensor]:
    """The parameters in native order `names`, checked for the kernels."""
    named = dict(model.named_parameters())
    if list(named) != names:
        head = "the linear classifier" if model.head is None else f"the '{model.head}' head"
        expects = ("the parameters of wekws/model/fsmn.py FSMN, in state_dict order" if label == "FSMN" else
                   f"the parameters of wekws/model/kws_model.py with the {label} backbone and {head}, in "
                   "named_parameters order")
        raise RuntimeError(f"wekws_b200: {label} training expects {expects} {names}; got {list(named)}")
    params = [named[n] for n in names]
    for n, p in zip(names, params):
        if p.device != dev or p.dtype != torch.float32 or not p.is_contiguous():
            raise ValueError(f"wekws_b200: {label} training needs every parameter as a contiguous float32 tensor on "
                             f"{dev}; {n} is {p.dtype} on {p.device}{'' if p.is_contiguous() else ', not contiguous'}")
    return params


def _buffers(model, dev: torch.device, bns: List[nn.BatchNorm1d], label: str):
    """(CMVN mean / istd or Nones, running statistics in native order, (momentum, eps) per BatchNorm, counters) of
    the BatchNorms `bns`."""
    running, hyper, counters = [], [], []
    for bn in bns:
        if not bn.track_running_stats or bn.running_mean is None or not bn.affine:
            raise ValueError(f"wekws_b200: {label} training needs affine BatchNorms that track running statistics")
        for t in (bn.running_mean, bn.running_var):
            if t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError(f"wekws_b200: {label} training needs the BatchNorm running statistics as contiguous "
                                 f"float32 tensors on {dev}")
        running += [bn.running_mean, bn.running_var]
        hyper += [float(bn.momentum), float(bn.eps)]
        counters.append(bn.num_batches_tracked)
    mean = istd = None
    if model.global_cmvn is not None:
        mean, istd = (t.to(device=dev, dtype=torch.float32).contiguous()
                      for t in (model.global_cmvn.mean, model.global_cmvn.istd))
    return (mean, istd), running, (C.c_double * len(hyper))(*hyper), counters


def _grad_out(g_out: torch.Tensor, dev: torch.device) -> torch.Tensor:
    if g_out.dtype != torch.float32 or g_out.device != dev:
        raise ValueError(f"wekws_b200: the logits' gradient must be float32 on {dev}, got {g_out.dtype} on "
                         f"{g_out.device}")
    return g_out.contiguous()


class _Config:
    """A config-only native model with its head (the batch-statistics entry points read nothing else from it),
    destroyed on exit.  `net` is (config, HEAD_* id)."""

    def __init__(self, net):
        cfg, head = net
        self.h = _native.create("wekws_model_create", C.byref(cfg))
        if head != _native.HEAD_LINEAR:
            _native.invoke("wekws_model_set_head", self.h, head)

    def __enter__(self):
        return self.h

    def __exit__(self, *exc):
        _native.lib().wekws_model_destroy(self.h)


def _run_forward(net, x, params, cmvn, running, hyper, drop, cache_shape, save: bool):
    """(logits, out_cache, saved activations -- empty without `save`) of the ``wekws_train_forward`` call: logits
    (B, T, odim), or (B, odim) with a head."""
    dev = x.device
    B, T = x.shape[0], x.shape[1]
    lib = _native.lib()
    cfg, head = net
    out = torch.empty((B, T, cfg.odim) if head == _native.HEAD_LINEAR else (B, cfg.odim), device=dev,
                      dtype=torch.float32)
    out_cache = torch.empty(cache_shape, device=dev, dtype=torch.float32)
    with _Config(net) as h:
        saved = torch.empty(int(lib.wekws_train_saved_floats(h, B, T)) if save else 0, device=dev, dtype=torch.float32)
        ws = torch.empty(int(lib.wekws_train_workspace_bytes(h, B, T, int(save))), device=dev, dtype=torch.uint8)
        _native.call("wekws_train_forward", h, x, _pointers(params), len(params), cmvn[0], cmvn[1],
                     _pointers(running), hyper, *drop, out, out_cache, saved if save else None, int(save), ws, B, T,
                     device=dev)
    return out, out_cache, saved


class _BatchStatsTrain(torch.autograd.Function):
    """(logits, out_cache) of an MDTC, MDTC with a head or TCN / DS-TCN training forward of the native model `net`
    (config, head id), whose Dropout arguments `drop` are (seed, probabilities, their count); the backward returns one
    gradient per parameter."""

    @staticmethod
    def forward(ctx, net, x, cmvn, running, hyper, drop, cache_shape, *params):
        out, out_cache, saved = _run_forward(net, x, params, cmvn, running, hyper, drop, cache_shape, True)
        kept = (out,) if net[0].backbone != _native.BACKBONE_MDTC else ()   # only the TCN backward reads the logits
        ctx.save_for_backward(x, saved, *kept, *params)  # the version check: no in-place change before backward
        ctx.net, ctx.cmvn, ctx.drop, ctx.nkept = net, cmvn, drop, len(kept)
        ctx.mark_non_differentiable(out_cache)
        return out, out_cache

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, _g_cache):
        x, saved, *rest = ctx.saved_tensors
        kept, params = rest[:ctx.nkept], rest[ctx.nkept:]
        dev = x.device
        B, T = x.shape[0], x.shape[1]
        g_out = _grad_out(g_out, dev)
        grads = [torch.empty_like(p) for p in params]
        with _Config(ctx.net) as h:
            ws = torch.empty(int(_native.lib().wekws_train_backward_workspace_bytes(h, B, T)), device=dev,
                             dtype=torch.uint8)
            _native.call("wekws_train_backward", h, x, _pointers(params), len(params), ctx.cmvn[0], ctx.cmvn[1],
                         saved, kept[0] if kept else None, g_out, *ctx.drop, B, T, _pointers(grads), ws, device=dev)
        return (None,) * 7 + tuple(grads)


def _load(model, dev: torch.device, params) -> C.c_void_p:
    """The model's native handle on `dev` with `params` packed into it (one launch)."""
    h = model._training_handle(dev)
    _native.call("wekws_model_load_params", h, _pointers(params), len(params), device=dev)
    return h


class _PackedTrain(torch.autograd.Function):
    """(logits, out_cache) of the FSMN or GRU training forward, which runs on the model's native handle with the
    parameters packed into it; the backward returns one gradient per parameter."""

    @staticmethod
    def forward(ctx, model, x, *params):
        dev = x.device
        B, T = x.shape[0], x.shape[1]
        out = torch.empty(B, T, model.odim, device=dev, dtype=torch.float32)
        if B > 0 and T > 0:
            h = _load(model, dev, params)
            out_cache = torch.empty(model.cache_shape(B), device=dev, dtype=torch.float32)
            saved = torch.empty(int(_native.lib().wekws_train_saved_floats(h, B, T)), device=dev, dtype=torch.float32)
            _native.call("wekws_model_train_forward", h, x, out, out_cache, saved, B, T, device=dev)
        else:
            h, saved = None, torch.empty(0, device=dev)
            out_cache = torch.zeros(model.cache_shape(B), device=dev, dtype=torch.float32)
        kept = (out,) if _kind(model) == "gru" else ()   # the Sigmoid backward reads the logits
        ctx.save_for_backward(x, saved, *kept, *params)  # the version check: no in-place change before backward
        ctx.model, ctx.handle, ctx.nkept = model, h, len(kept)
        ctx.mark_non_differentiable(out_cache)
        return out, out_cache

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, _g_cache):
        x, saved, *rest = ctx.saved_tensors
        kept, params = rest[:ctx.nkept], rest[ctx.nkept:]
        grads = [torch.empty_like(p) for p in params]
        B, T = x.shape[0], x.shape[1]
        if B == 0 or T == 0:
            for g in grads:
                g.zero_()
            return (None, None) + tuple(grads)
        dev = x.device
        model = ctx.model
        h = model.__dict__.get("_handle")
        if h is not ctx.handle or model._handle_dev != dev:
            h = _load(model, dev, params)             # the handle was rebuilt since the forward: same values again
        g_out = _grad_out(g_out, dev)
        ws = torch.empty(int(_native.lib().wekws_train_backward_workspace_bytes(h, B, T)), device=dev,
                         dtype=torch.uint8)
        _native.call("wekws_model_backward", h, x, saved, kept[0] if kept else None, g_out, B, T, _pointers(grads),
                     len(grads), ws, device=dev)
        return (None, None) + tuple(grads)


def forward(model, x: torch.Tensor, in_cache: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The training forward of `model` (after ``route`` returned True, with ``x`` checked as (B, T, idim) float32 on
    CUDA)."""
    dev = x.device
    bb = model.backbone
    kind = _kind(model)
    if kind in ("fsmn", "gru"):
        label = _label(kind)
        _check_inputs(x, in_cache, label, "with grad is not supported -- pass no in_cache, or call under "
                      "torch.no_grad()")
        names = fsmn_train.param_names(bb.fsmn_layers) if kind == "fsmn" else gru_train.param_names(bb.num_layers)
        params = _params(model, dev, names, label)
        return _PackedTrain.apply(model, x.contiguous(), *params)
    label = _label(bb.kind)
    head = _native.HEAD_LINEAR
    if bb.kind == "mdtc" and model.head is not None:
        names = mdtc_train.head_param_names(bb.num_stack, bb.stack_size)
        head = {"global": _native.HEAD_GLOBAL, "last": _native.HEAD_LAST}[model.head]
    elif bb.kind == "mdtc":
        names = mdtc_train.param_names(bb.num_stack, bb.stack_size)
    else:
        names = tcn_train.param_names(bb.num_layers, bb.ds)
    params = _params(model, dev, names, label)
    cmvn, running, hyper, counters = _buffers(model, dev, _batch_norms(model), label)
    net = (model._native_config(), head)
    x = x.contiguous()
    seed, ps = 0, []                             # Dropout: none in MDTC, one in a head, one per TCN block
    if bb.kind != "mdtc":
        seed, ps = tcn_train.draw_dropout(model)
    elif head != _native.HEAD_LINEAR:
        seed, p = mdtc_train.draw_head_dropout(model)
        ps = [p]
    drop = (seed, (C.c_double * len(ps))(*ps), len(ps))
    B = x.shape[0]
    if wants_grad(model):
        out, out_cache = _BatchStatsTrain.apply(net, x, cmvn, running, hyper, drop, model.cache_shape(B), *params)
    else:
        out, out_cache, _ = _run_forward(net, x, params, cmvn, running, hyper, drop, model.cache_shape(B), False)
    torch._foreach_add_(counters, 1)
    model.invalidate()           # the running statistics changed without a version-counter bump: repack for eval
    return out, out_cache
