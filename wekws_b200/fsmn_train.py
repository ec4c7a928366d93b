"""Training the FSMN model on the device: the training-mode forward and its backward for ``Executor.train``.

After ``model.train()``, with grad mode on and a parameter requiring grad, an FSMN ``KWSModel`` returns logits attached
to the autograd graph; ``loss.backward()`` then fills ``.grad`` of every parameter of the reference's FSMN
(wekws/model/fsmn.py).  The forward is the fused kernel of csrc/fsmn.cu in its storing instantiation (its logits are
the eval logits, bit for bit: the FSMN has no BatchNorm, and its Dropout is never called), the backward the kernels of
csrc/fsmn_grad.cu.  Each forward first packs the parameters' current values into the native model on the device (one
launch), so ``optimizer.step()`` needs no host round trip.

Not supported, and refused: a streaming cache with grad, features that require grad, and double backward.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Tuple

import torch
from torch.autograd.function import once_differentiable

from . import _native


def param_names(num_layers: int) -> List[str]:
    """The parameter order of the native entry points: the FSMN model's ``state_dict`` order without its buffers."""
    names = ["backbone.in_linear1.linear.weight", "backbone.in_linear1.linear.bias",
             "backbone.in_linear2.linear.weight", "backbone.in_linear2.linear.bias"]
    for l in range(num_layers):
        p = f"backbone.fsmn.{l}."
        names += [p + "0.linear.weight", p + "1.conv_left.weight", p + "1.conv_right.weight",
                  p + "2.linear.weight", p + "2.linear.bias"]
    return names + ["backbone.out_linear1.linear.weight", "backbone.out_linear1.linear.bias",
                    "backbone.out_linear2.linear.weight", "backbone.out_linear2.linear.bias"]


def saved_floats_per_frame(bb) -> int:
    """Activations the training forward keeps per frame: in_linear1 and in_linear2 outputs, per layer the projection,
    the memory-block output and the layer output, and the out_linear1 output."""
    return bb.input_affine_dim + bb.linear_dim + bb.fsmn_layers * (2 * bb.proj_dim + bb.linear_dim) + bb.output_affine_dim


def _pointers(tensors) -> C.Array:
    return (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _params(model, dev: torch.device) -> List[torch.Tensor]:
    named = dict(model.named_parameters())
    names = param_names(model.backbone.fsmn_layers)
    if list(named) != names:
        raise RuntimeError("wekws_b200: FSMN training expects the parameters of wekws/model/fsmn.py FSMN, in state_dict "
                           f"order {names}; got {list(named)}")
    params = [named[n] for n in names]
    for n, p in zip(names, params):
        if p.device != dev or p.dtype != torch.float32 or not p.is_contiguous():
            raise ValueError(f"wekws_b200: FSMN training needs every parameter as a contiguous float32 tensor on "
                             f"{dev}; {n} is {p.dtype} on {p.device}{'' if p.is_contiguous() else ', not contiguous'}")
    return params


def _load(model, dev: torch.device, params) -> C.c_void_p:
    """The model's native handle on `dev` with `params` packed into it (one launch)."""
    h = model._training_handle(dev)
    _native.call("wekws_fsmn_load_params", h, _pointers(params), len(params), device=dev)
    return h


class _FsmnTrain(torch.autograd.Function):
    """(logits, out_cache) of the training forward; the backward returns one gradient per parameter."""

    @staticmethod
    def forward(ctx, model, x, *params):
        dev = x.device
        B, T = x.shape[0], x.shape[1]
        out = torch.empty(B, T, model.odim, device=dev, dtype=torch.float32)
        if B > 0 and T > 0:
            h = _load(model, dev, params)
            out_cache = torch.empty(model.cache_shape(B), device=dev, dtype=torch.float32)
            saved = torch.empty(int(_native.lib().wekws_fsmn_train_saved_floats(h, B, T)), device=dev,
                                dtype=torch.float32)
            _native.call("wekws_fsmn_train_forward", h, x, out, out_cache, saved, B, T, device=dev)
        else:
            h, saved = None, torch.empty(0, device=dev)
            out_cache = torch.zeros(model.cache_shape(B), device=dev, dtype=torch.float32)
        ctx.save_for_backward(x, saved, *params)      # the version check: no in-place change before backward
        ctx.model, ctx.handle = model, h
        ctx.mark_non_differentiable(out_cache)
        return out, out_cache

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, _g_cache):
        x, saved, *params = ctx.saved_tensors
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
        if g_out.dtype != torch.float32 or g_out.device != dev:
            raise ValueError(f"wekws_b200: the logits' gradient must be float32 on {dev}, got {g_out.dtype} on "
                             f"{g_out.device}")
        g_out = g_out.contiguous()
        ws = torch.empty(int(_native.lib().wekws_fsmn_backward_workspace_bytes(h, B, T)), device=dev,
                         dtype=torch.uint8)
        _native.call("wekws_fsmn_backward", h, x, saved, g_out, B, T, _pointers(grads), len(grads), ws, device=dev)
        return (None, None) + tuple(grads)


def wants_grad(model) -> bool:
    """True when a training-mode call must build the autograd graph: grad mode on, a parameter requiring grad."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters())


def forward(model, x: torch.Tensor, in_cache: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The training forward of an FSMN ``KWSModel`` (``x`` already checked as (B, T, idim) float32 on CUDA)."""
    if in_cache is not None and in_cache.numel() > 0:
        raise ValueError("wekws_b200: FSMN training runs from empty caches (as Executor.train does); a streaming cache "
                         "with grad is not supported -- pass no in_cache, or call under torch.no_grad()")
    if x.requires_grad:
        raise ValueError("wekws_b200: FSMN training computes parameter gradients only; features that require grad "
                         "are not supported (detach them)")
    params = _params(model, x.device)
    return _FsmnTrain.apply(model, x.contiguous(), *params)
