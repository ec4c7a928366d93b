"""Training the TCN / DS-TCN models on the device: the batch-statistics forward with device Dropout masks, and its
backward, for ``Executor.train``.

After ``model.enable_training(device_dropout=True)`` and ``model.train()``, a TCN or DS-TCN ``KWSModel`` with the
per-frame linear classifier runs the training-mode forward of the reference's wekws/model/tcn.py: every BatchNorm as
in MDTC training (mdtc_train.py), and every block's ``nn.Dropout`` applying a mask made on the device.  No device
generator reproduces torch's Bernoulli stream, so the mask is a documented pure function of a 64-bit seed
(include/wekws_b200.h, ``wekws_tcn_train_forward``), and the seed is one draw from torch's default CPU generator per
training forward (``frontend.draw_seed``): ``torch.manual_seed`` makes a run reproducible.  When every block's ``p``
is 0 nothing is drawn.  ``p`` is read from each block's own ``nn.Dropout`` at call time.  The backward recomputes the
masks from the seed; they are never stored.

Refused as in MDTC training: a non-empty streaming cache, features that require grad, ``forward_softmax``,
``momentum=None``, non-contiguous or non-float32 parameters, and double backward.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Tuple

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _native, mdtc_train
from .frontend import draw_seed

HIDDEN, MAX_K, MAX_LAYERS, MAX_IDIM, MAX_ODIM = (64, 256), 8, 8, 128, 4096


def param_names(num_layers: int, ds: bool) -> List[str]:
    """The parameter order of the native entry points: the TCN / DS-TCN model's ``named_parameters()`` order."""
    names = ["preprocessing.out.0.weight", "preprocessing.out.0.bias"]
    for l in range(num_layers):
        for j in ((0, 1, 3, 4) if ds else (0, 1)):
            names += [f"backbone.network.{l}.cnn.{j}.weight", f"backbone.network.{l}.cnn.{j}.bias"]
    return names + ["classifier.linear.weight", "classifier.linear.bias"]


def _name(model) -> str:
    return "DS-TCN" if model.backbone.ds else "TCN"


def batch_norms(model) -> List[nn.BatchNorm1d]:
    """Every BatchNorm in the order of the native entry points: cnn.1 [, cnn.4] of each block."""
    return [blk.cnn[j] for blk in model.backbone.network for j in ((1, 4) if model.backbone.ds else (1,))]


def dropouts(model) -> List[nn.Dropout]:
    """Every block's Dropout, in block order."""
    return [blk.cnn[-1] for blk in model.backbone.network]


def saved_floats(num_layers: int, hdim: int, ds: bool, B: int, T: int) -> int:
    """Floats the grad-mode forward keeps: each BatchNorm's mean and invstd (as doubles), the preprocessing output,
    per block its pre-BatchNorm tensors and its output."""
    nbn = (2 if ds else 1) * num_layers
    return 4 * nbn * hdim + B * T * hdim * (1 + num_layers * (3 if ds else 2))


def forward_launches(num_layers: int, ds: bool) -> int:
    """Preprocessing; per block the depthwise conv and the pointwise GEMM (ds) or the conv GEMM (dense); classifier."""
    return 2 + (2 if ds else 1) * num_layers


def backward_launches(num_layers: int, ds: bool) -> int:
    """Classifier input gradient and weight gradient; per block the input gradient GEMM and weight-gradient GEMM (and
    the depthwise backward, ds); the preprocessing weight gradient; the ordered sum of the partials."""
    return 4 + (3 if ds else 2) * num_layers


def check_trainable(model) -> None:
    """Raises NotImplementedError unless `model` is a TCN / DS-TCN configuration the training kernels run."""
    bb = model.backbone
    name = _name(model)
    if model.head is not None:
        raise NotImplementedError(f"wekws_b200: {name} training runs with the per-frame linear classifier; the "
                                  f"'{model.head}' head has Dropout, which is not implemented")
    if not isinstance(model.activation, (nn.Sigmoid, nn.Identity)):
        raise NotImplementedError(f"wekws_b200: {name} training needs the Sigmoid or Identity activation")
    if model.hdim not in HIDDEN or not 2 <= bb.kernel_size <= MAX_K or not 1 <= bb.num_layers <= MAX_LAYERS \
            or model.idim > MAX_IDIM or model.odim > MAX_ODIM:
        raise NotImplementedError(f"wekws_b200: {name} training supports hidden_dim 64 or 256, kernel_size 2..{MAX_K}, "
                                  f"1..{MAX_LAYERS} layers, input_dim <= {MAX_IDIM} and output_dim <= {MAX_ODIM}; "
                                  f"got hidden {model.hdim}, kernel {bb.kernel_size}, {bb.num_layers} layers, input "
                                  f"{model.idim}, output {model.odim}")


def check_call(model, x: torch.Tensor, in_cache: torch.Tensor) -> None:
    """The refusals that need no device (mdtc_train.check_call, for this model's BatchNorms)."""
    mdtc_train.check_call(model, x, in_cache, batch_norms(model), _name(model))


def _dropout(model) -> Tuple[int, C.Array]:
    """(seed, per-block p as host doubles): one draw from torch's default generator when any p > 0, else seed 0."""
    ps = [float(d.p) for d in dropouts(model)]
    seed = draw_seed() if any(p > 0 for p in ps) else 0
    return seed, (C.c_double * len(ps))(*ps)


def _run_forward(cfg, x, params, cmvn, running, hyper, drop, cache_shape, save: bool):
    """(logits, out_cache, saved activations -- empty without `save`)."""
    dev = x.device
    B, T = x.shape[0], x.shape[1]
    lib = _native.lib()
    out = torch.empty(B, T, cfg.odim, device=dev, dtype=torch.float32)
    out_cache = torch.empty(cache_shape, device=dev, dtype=torch.float32)
    with mdtc_train._Config(cfg) as h:
        saved = torch.empty(int(lib.wekws_tcn_train_saved_floats(h, B, T)) if save else 0, device=dev,
                            dtype=torch.float32)
        ws = torch.empty(int(lib.wekws_tcn_train_workspace_bytes(h, B, T, int(save))), device=dev, dtype=torch.uint8)
        _native.call("wekws_tcn_train_forward", h, x, mdtc_train._pointers(params), len(params), cmvn[0], cmvn[1],
                     mdtc_train._pointers(running), hyper, drop[0], drop[1], out, out_cache,
                     saved if save else None, int(save), ws, B, T, device=dev)
    return out, out_cache, saved


class _TcnTrain(torch.autograd.Function):
    """(logits, out_cache) of the training forward; the backward returns one gradient per parameter."""

    @staticmethod
    def forward(ctx, cfg, x, cmvn, running, hyper, drop, cache_shape, *params):
        out, out_cache, saved = _run_forward(cfg, x, params, cmvn, running, hyper, drop, cache_shape, True)
        ctx.save_for_backward(x, saved, out, *params)  # the version check: no in-place change before backward
        ctx.cfg, ctx.cmvn, ctx.drop = cfg, cmvn, drop
        ctx.mark_non_differentiable(out_cache)
        return out, out_cache

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, _g_cache):
        x, saved, out, *params = ctx.saved_tensors
        dev = x.device
        B, T = x.shape[0], x.shape[1]
        if g_out is None:
            g_out = torch.zeros(B, T, ctx.cfg.odim, device=dev, dtype=torch.float32)
        if g_out.dtype != torch.float32 or g_out.device != dev:
            raise ValueError(f"wekws_b200: the logits' gradient must be float32 on {dev}, got {g_out.dtype} on "
                             f"{g_out.device}")
        g_out = g_out.contiguous()
        grads = [torch.empty_like(p) for p in params]
        with mdtc_train._Config(ctx.cfg) as h:
            ws = torch.empty(int(_native.lib().wekws_tcn_backward_workspace_bytes(h, B, T)), device=dev,
                             dtype=torch.uint8)
            _native.call("wekws_tcn_backward", h, x, mdtc_train._pointers(params), len(params), ctx.cmvn[0],
                         ctx.cmvn[1], saved, out, g_out, ctx.drop[0], ctx.drop[1], B, T, mdtc_train._pointers(grads),
                         ws, device=dev)
        return (None,) * 7 + tuple(grads)


def forward(model, x: torch.Tensor, in_cache: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The training forward of a TCN / DS-TCN ``KWSModel`` (``x`` already checked as (B, T, idim) float32 on CUDA,
    and by ``check_call``)."""
    B = x.shape[0]
    dev = x.device
    bb = model.backbone
    params = mdtc_train._params(model, dev, param_names(bb.num_layers, bb.ds), _name(model))
    cmvn, running, hyper, counters = mdtc_train._buffers(model, dev, batch_norms(model), _name(model))
    cfg = model._native_config()
    x = x.contiguous()
    drop = _dropout(model)
    if mdtc_train.wants_grad(model):
        out, out_cache = _TcnTrain.apply(cfg, x, cmvn, running, hyper, drop, model.cache_shape(B), *params)
    else:
        out, out_cache, _ = _run_forward(cfg, x, params, cmvn, running, hyper, drop, model.cache_shape(B), False)
    torch._foreach_add_(counters, 1)
    model.invalidate()           # the running statistics changed without a version-counter bump: repack for eval
    return out, out_cache
