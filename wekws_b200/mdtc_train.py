"""Training the MDTC model on the device: the batch-statistics forward and its backward for ``Executor.train``.

After ``model.enable_training()`` and ``model.train()``, an MDTC ``KWSModel`` with the per-frame linear classifier
runs the training-mode forward of the reference's wekws/model/kws_model.py: every BatchNorm normalises with the biased
variance of the batch (all B * T frames, padding included), updates ``running_mean`` / ``running_var`` (the latter with
the unbiased variance) with its own ``momentum`` and ``eps``, and counts ``num_batches_tracked``.  With grad mode on
and a parameter requiring grad the logits are attached to the autograd graph, and ``loss.backward()`` fills ``.grad``
of every parameter; otherwise the same forward runs without keeping activations.  The kernels are those of
csrc/mdtc_train.cu; they read the parameters, the CMVN buffers and the running statistics where they live on the
device, so ``optimizer.step()`` needs no host round trip.  The running statistics are written by a kernel, behind the
version counters' back, so each training forward marks the packed eval model stale: the next eval call repacks.

The opt-in exists because a BatchNorm model in training mode gives other outputs than in eval mode and overwrites its
running statistics: a model left in ``train()`` by accident keeps refusing to run.  The MDTC backbone has no Dropout;
the TCN / DS-TCN backbones train through tcn_train.py, and the ``global`` / ``last`` heads are not supported.

Refused: a non-empty streaming cache, features that require grad, ``forward_softmax``, ``momentum=None``, non-contiguous
or non-float32 parameters, and double backward.
"""
from __future__ import annotations

import ctypes as C
from typing import List, Tuple

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _native

_BLOCK_PARAMS = ["conv1.conv.weight", "conv1.conv.bias", "conv1.bn.weight", "conv1.bn.bias", "conv1.pointwise.weight",
                 "conv1.pointwise.bias", "bn1.weight", "bn1.bias", "conv2.weight", "conv2.bias", "bn2.weight",
                 "bn2.bias"]
MAX_BLOCKS, MAX_K, MAX_IDIM, MAX_ODIM = 25, 8, 128, 16


def block_prefixes(num_stack: int, stack_size: int) -> List[str]:
    """The MDTC blocks in execution order: the preprocessor, then each stack's res_blocks."""
    return ["backbone.preprocessor"] + [f"backbone.blocks.{s}.res_blocks.{l}" for s in range(num_stack)
                                        for l in range(stack_size)]


def param_names(num_stack: int, stack_size: int) -> List[str]:
    """The parameter order of the native entry points: the MDTC model's ``named_parameters()`` order."""
    names = ["preprocessing.out.0.weight", "preprocessing.out.0.bias"]
    for p in block_prefixes(num_stack, stack_size):
        names += [f"{p}.{n}" for n in _BLOCK_PARAMS]
    return names + ["classifier.linear.weight", "classifier.linear.bias"]


def saved_floats(num_blocks: int, hdim: int, B: int, T: int) -> int:
    """Floats the grad-mode forward keeps: each BatchNorm's mean and invstd (as doubles), the preprocessing output,
    per block its three pre-BatchNorm tensors and its output, and the sum of the stack outputs."""
    return 12 * num_blocks * hdim + B * T * hdim * (4 * num_blocks + 2)


def forward_launches(num_blocks: int) -> int:
    """Preprocessing; per block the depthwise conv and the two pointwise convs; the stack sum and classifier."""
    return 2 + 3 * num_blocks


def backward_launches(num_blocks: int) -> int:
    """Classifier; per block BN2's gradient statistics, conv2, pointwise and depthwise; preprocessing; slice sums."""
    return 3 + 4 * num_blocks


def check_trainable(model) -> None:
    """Raises NotImplementedError unless `model` is a configuration the training kernels run."""
    bb = model.backbone
    kind = "gru" if isinstance(bb, nn.GRU) else getattr(bb, "kind", None)
    if kind in ("tcn", "ds_tcn"):
        raise NotImplementedError(f"wekws_b200: training the {kind.upper().replace('_', '-')} backbone applies Dropout "
                                  "masks made on the device, not torch's Bernoulli draws: opt in with "
                                  "model.enable_training(device_dropout=True)")
    if kind != "mdtc":
        raise NotImplementedError(f"wekws_b200: training is not implemented for the {str(kind).upper()} backbone")
    if model.head is not None:
        raise NotImplementedError(f"wekws_b200: MDTC training runs with the per-frame linear classifier; the "
                                  f"'{model.head}' head has Dropout, which is not implemented")
    if not isinstance(model.activation, (nn.Sigmoid, nn.Identity)):
        raise NotImplementedError("wekws_b200: MDTC training needs the Sigmoid or Identity activation")
    L = 1 + bb.num_stack * bb.stack_size
    if model.hdim not in (32, 64) or bb.kernel_size > MAX_K or model.idim > MAX_IDIM or model.odim > MAX_ODIM \
            or L > MAX_BLOCKS:
        raise NotImplementedError(f"wekws_b200: MDTC training supports hidden_dim 32 or 64, kernel_size <= {MAX_K}, "
                                  f"input_dim <= {MAX_IDIM}, output_dim <= {MAX_ODIM} and at most {MAX_BLOCKS} blocks; "
                                  f"got hidden {model.hdim}, kernel {bb.kernel_size}, input {model.idim}, output "
                                  f"{model.odim}, {L} blocks")


def batch_norms(model) -> List[nn.BatchNorm1d]:
    """Every BatchNorm in the order of the native entry points: conv1.bn, bn1, bn2 of each block."""
    bb = model.backbone
    blocks = [bb.preprocessor] + [blk for st in bb.blocks for blk in st.res_blocks]
    return [m for blk in blocks for m in (blk.conv1.bn, blk.bn1, blk.bn2)]


def _pointers(tensors) -> C.Array:
    return (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _params(model, dev: torch.device, names: List[str] = None, what: str = "MDTC") -> List[torch.Tensor]:
    """The parameters in native order (``names``, default the MDTC order), checked for the kernels."""
    named = dict(model.named_parameters())
    if names is None:
        names = param_names(model.backbone.num_stack, model.backbone.stack_size)
    if list(named) != names:
        raise RuntimeError(f"wekws_b200: {what} training expects the parameters of wekws/model/kws_model.py with the "
                           f"{what} backbone and the linear classifier, in named_parameters order {names}; got "
                           f"{list(named)}")
    params = [named[n] for n in names]
    for n, p in zip(names, params):
        if p.device != dev or p.dtype != torch.float32 or not p.is_contiguous():
            raise ValueError(f"wekws_b200: {what} training needs every parameter as a contiguous float32 tensor on "
                             f"{dev}; {n} is {p.dtype} on {p.device}{'' if p.is_contiguous() else ', not contiguous'}")
    return params


def _buffers(model, dev: torch.device, bns: List[nn.BatchNorm1d] = None, what: str = "MDTC"):
    """(CMVN mean / istd or Nones, running statistics in native order, (momentum, eps) per BatchNorm, counters) of
    the BatchNorms ``bns`` (default the MDTC ones)."""
    running, hyper, counters = [], [], []
    for bn in batch_norms(model) if bns is None else bns:
        if not bn.track_running_stats or bn.running_mean is None or not bn.affine:
            raise ValueError(f"wekws_b200: {what} training needs affine BatchNorms that track running statistics")
        for t in (bn.running_mean, bn.running_var):
            if t.device != dev or t.dtype != torch.float32 or not t.is_contiguous():
                raise ValueError(f"wekws_b200: {what} training needs the BatchNorm running statistics as contiguous "
                                 f"float32 tensors on {dev}")
        running += [bn.running_mean, bn.running_var]
        hyper += [float(bn.momentum), float(bn.eps)]
        counters.append(bn.num_batches_tracked)
    mean = istd = None
    if model.global_cmvn is not None:
        mean, istd = (t.to(device=dev, dtype=torch.float32).contiguous()
                      for t in (model.global_cmvn.mean, model.global_cmvn.istd))
    return (mean, istd), running, (C.c_double * len(hyper))(*hyper), counters


class _Config:
    """A config-only native model (the training entry points read nothing else from it), destroyed on exit."""

    def __init__(self, cfg: _native.ModelConfig):
        self.h = _native.create("wekws_model_create", C.byref(cfg))

    def __enter__(self):
        return self.h

    def __exit__(self, *exc):
        _native.lib().wekws_model_destroy(self.h)


def _run_forward(cfg, x, params, cmvn, running, hyper, cache_shape, save: bool):
    """(logits, out_cache, saved activations -- empty without `save`)."""
    dev = x.device
    B, T = x.shape[0], x.shape[1]
    lib = _native.lib()
    out = torch.empty(B, T, cfg.odim, device=dev, dtype=torch.float32)
    out_cache = torch.empty(cache_shape, device=dev, dtype=torch.float32)
    with _Config(cfg) as h:
        saved = torch.empty(int(lib.wekws_mdtc_train_saved_floats(h, B, T)) if save else 0, device=dev,
                            dtype=torch.float32)
        ws = torch.empty(int(lib.wekws_mdtc_train_workspace_bytes(h, B, T, int(save))), device=dev, dtype=torch.uint8)
        _native.call("wekws_mdtc_train_forward", h, x, _pointers(params), len(params), cmvn[0], cmvn[1],
                     _pointers(running), hyper, out, out_cache, saved if save else None, int(save), ws, B, T,
                     device=dev)
    return out, out_cache, saved


class _MdtcTrain(torch.autograd.Function):
    """(logits, out_cache) of the training forward; the backward returns one gradient per parameter."""

    @staticmethod
    def forward(ctx, cfg, x, cmvn, running, hyper, cache_shape, *params):
        out, out_cache, saved = _run_forward(cfg, x, params, cmvn, running, hyper, cache_shape, True)
        ctx.save_for_backward(x, saved, *params)      # the version check: no in-place change before backward
        ctx.cfg, ctx.cmvn = cfg, cmvn
        ctx.mark_non_differentiable(out_cache)
        return out, out_cache

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, _g_cache):
        x, saved, *params = ctx.saved_tensors
        dev = x.device
        B, T = x.shape[0], x.shape[1]
        if g_out is None:
            g_out = torch.zeros(B, T, ctx.cfg.odim, device=dev, dtype=torch.float32)
        if g_out.dtype != torch.float32 or g_out.device != dev:
            raise ValueError(f"wekws_b200: the logits' gradient must be float32 on {dev}, got {g_out.dtype} on "
                             f"{g_out.device}")
        g_out = g_out.contiguous()
        grads = [torch.empty_like(p) for p in params]
        with _Config(ctx.cfg) as h:
            ws = torch.empty(int(_native.lib().wekws_mdtc_backward_workspace_bytes(h, B, T)), device=dev,
                             dtype=torch.uint8)
            _native.call("wekws_mdtc_backward", h, x, _pointers(params), len(params), ctx.cmvn[0], ctx.cmvn[1], saved,
                         g_out, B, T, _pointers(grads), ws, device=dev)
        return (None,) * 6 + tuple(grads)


def wants_grad(model) -> bool:
    """True when a training-mode call must build the autograd graph: grad mode on, a parameter requiring grad."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in model.parameters())


def check_call(model, x: torch.Tensor, in_cache: torch.Tensor, bns: List[nn.BatchNorm1d] = None,
               what: str = "MDTC") -> None:
    """The refusals that need no device: a streaming cache, features that require grad, a batch of one frame (torch's
    own error), a BatchNorm (of ``bns``, default the MDTC ones) with momentum=None."""
    if in_cache is not None and in_cache.numel() > 0:
        raise ValueError(f"wekws_b200: {what} training runs from empty caches (as Executor.train does); a streaming "
                         "cache is not supported in training mode -- pass no in_cache, or call model.eval()")
    if x.requires_grad:
        raise ValueError(f"wekws_b200: {what} training computes parameter gradients only; features that require grad "
                         "are not supported (detach them)")
    if x.dim() == 3 and x.shape[0] * x.shape[1] <= 1:
        raise ValueError("Expected more than 1 value per channel when training, got input size "
                         f"{torch.Size([x.shape[0], model.hdim, x.shape[1]])}")
    for bn in batch_norms(model) if bns is None else bns:
        if bn.momentum is None:
            raise ValueError("wekws_b200: BatchNorm momentum=None (a cumulative moving average) is not supported in "
                             f"{what} training; set a momentum")


def forward(model, x: torch.Tensor, in_cache: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The training forward of an MDTC ``KWSModel`` (``x`` already checked as (B, T, idim) float32 on CUDA, and by
    ``check_call``)."""
    B, T = x.shape[0], x.shape[1]
    dev = x.device
    params = _params(model, dev)
    cmvn, running, hyper, counters = _buffers(model, dev)
    cfg = model._native_config()
    x = x.contiguous()
    if wants_grad(model):
        out, out_cache = _MdtcTrain.apply(cfg, x, cmvn, running, hyper, model.cache_shape(B), *params)
    else:
        out, out_cache, _ = _run_forward(cfg, x, params, cmvn, running, hyper, model.cache_shape(B), False)
    torch._foreach_add_(counters, 1)
    model.invalidate()           # the running statistics changed without a version-counter bump: repack for eval
    return out, out_cache
