"""The training step's optimiser on the device: drop-ins for the two calls of wekws/utils/executor.py Executor.train
that follow loss.backward(),

    grad_norm = clip_grad_norm_(model.parameters(), clip)      # torch.nn.utils.clip_grad_norm_, norm_type 2
    optimizer.step()                                           # torch.optim.Adam(model.parameters(), **optim_conf)

run as csrc/optim.cu's kernels: the norm and the clip in two launches, the Adam update in one, each taking the
tensors as a table of pointers in its kernel parameters.  Neither call synchronises with the device or allocates
host-pinned or device memory beyond torch's caching allocator, so the host cost of a step is one pass over the
parameter list.  The rounding of every intermediate is written out in include/wekws_b200.h.

``Adam`` keeps torch.optim.Adam's arguments, defaults, param groups and state layout (``step`` a 0-dim float32 CPU
tensor, ``exp_avg`` / ``exp_avg_sq`` zeros_like(p)), so its state_dict() loads into torch.optim.Adam and back, and
ReduceLROnPlateau's lr changes apply on the next step.  Differences from torch: ``clip_grad_norm_`` sums the squares
in double (torch sums each tensor's in float32); it refuses a NaN ``max_norm``, which would make every torch gradient
NaN.  What the kernels do not implement is refused with NotImplementedError naming it, never run another way.
"""
from __future__ import annotations

import ctypes as C
import math
import types
import warnings

import torch

from . import _native

_REFUSED_FLAGS = (("amsgrad", False), ("maximize", False), ("capturable", False), ("differentiable", False),
                  ("decoupled_weight_decay", False))


_ONE = torch.tensor(1.0)


def adam_scalars(lr: float, beta1: float, beta2: float, step: float):
    """(step_size, bc2_sqrt) of one tensor at its ``step``: torch's _multi_tensor_adam expressions, in double."""
    bias_correction1 = 1 - beta1 ** step
    bias_correction2 = 1 - beta2 ** step
    return (lr / bias_correction1) * -1, bias_correction2 ** 0.5


def _check_tensor(t: torch.Tensor, what: str, device=None) -> None:
    """The layout the kernels read: dense, contiguous, float32 on a CUDA device (``device`` when given)."""
    if t.layout != torch.strided:
        raise NotImplementedError(f"wekws_b200 optimiser: {what} is {t.layout} (sparse); only dense tensors")
    if t.is_complex():
        raise NotImplementedError(f"wekws_b200 optimiser: {what} is complex ({t.dtype}); only float32")
    if t.dtype != torch.float32:
        raise NotImplementedError(f"wekws_b200 optimiser: {what} is {t.dtype}; only float32")
    if not t.is_cuda:
        raise NotImplementedError(f"wekws_b200 optimiser: {what} is on {t.device}; the step runs on CUDA (sm_90a) only")
    if device is not None and t.device != device:
        raise NotImplementedError(f"wekws_b200 optimiser: {what} is on {t.device}, another on {device}; "
                                  "mixed devices are not supported")
    if not t.is_contiguous():
        raise NotImplementedError(f"wekws_b200 optimiser: {what} is not contiguous")


def _pointers(tensors) -> C.Array:
    return (C.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])


def _numels(tensors) -> C.Array:
    return (C.c_int64 * len(tensors))(*[t.numel() for t in tensors])


class Adam(torch.optim.Optimizer):
    """torch.optim.Adam (L2 ``weight_decay``) whose step is one native launch per 512 parameter tensors.

    Refused with NotImplementedError: ``amsgrad``, ``maximize``, ``capturable``, ``differentiable``, ``fused=True``,
    ``decoupled_weight_decay=True``, a tensor ``lr`` or ``betas``, and parameters that are sparse, complex, not
    float32, not contiguous, on the CPU or on more than one device.  ``foreach`` is accepted and kept in the param
    groups, as torch does; it selects nothing here."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *,
                 foreach=None, maximize=False, capturable=False, differentiable=False, fused=None,
                 decoupled_weight_decay=False):
        if isinstance(lr, torch.Tensor):
            raise NotImplementedError("wekws_b200.Adam: a tensor lr is not supported; pass a float")
        if any(isinstance(b, torch.Tensor) for b in betas):
            raise NotImplementedError("wekws_b200.Adam: tensor betas are not supported; pass floats")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = {"lr": lr, "betas": tuple(betas), "eps": eps, "weight_decay": weight_decay, "amsgrad": amsgrad,
                    "maximize": maximize, "foreach": foreach, "capturable": capturable,
                    "differentiable": differentiable, "fused": fused,
                    "decoupled_weight_decay": decoupled_weight_decay}
        self._device = None
        super().__init__(params, defaults)

    @staticmethod
    def _check_group(group) -> None:
        for key, allowed in _REFUSED_FLAGS:
            if group[key] != allowed:
                raise NotImplementedError(f"wekws_b200.Adam: {key}={group[key]!r} is not supported")
        if group["fused"]:
            raise NotImplementedError("wekws_b200.Adam: fused=True is not supported (the step is already one launch)")
        if isinstance(group["lr"], torch.Tensor):
            raise NotImplementedError("wekws_b200.Adam: a tensor lr is not supported; pass a float")
        if any(isinstance(b, torch.Tensor) for b in group["betas"]):
            raise NotImplementedError("wekws_b200.Adam: tensor betas are not supported; pass floats")

    def add_param_group(self, param_group) -> None:
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        try:
            self._check_group(group)
            device = self._device
            for i, p in enumerate(group["params"]):
                _check_tensor(p, f"parameter {i} of group {len(self.param_groups) - 1}", device)
                device = p.device
        except (NotImplementedError, ValueError):
            self.param_groups.pop()
            raise
        self._device = device

    def load_state_dict(self, state_dict) -> None:
        super().load_state_dict(state_dict)
        for group in self.param_groups:
            self._check_group(group)
            for p in group["params"]:
                st = self.state.get(p)
                if st:
                    for key in ("exp_avg", "exp_avg_sq"):
                        _check_tensor(st[key], f"state {key!r}", p.device)
                        if st[key].shape != p.shape:
                            raise ValueError(f"wekws_b200.Adam: state {key!r} has shape {tuple(st[key].shape)}, "
                                             f"its parameter {tuple(p.shape)}")

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            self._check_group(group)
            params, grads, exp_avgs, exp_avg_sqs, steps = [], [], [], [], []
            for p in group["params"]:
                g = p.grad
                if g is None:
                    continue
                if g.is_sparse:
                    raise RuntimeError("Adam does not support sparse gradients, please consider SparseAdam instead")
                if g.dtype is not torch.float32 or g.get_device() != p.get_device() or not g.is_contiguous():
                    _check_tensor(g, "a gradient", p.device)
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = torch.tensor(0.0, dtype=torch.float32)
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                params.append(p)
                grads.append(g)
                exp_avgs.append(state["exp_avg"])
                exp_avg_sqs.append(state["exp_avg_sq"])
                steps.append(state["step"])
            if not params:
                continue
            torch._foreach_add_(steps, _ONE, alpha=1.0)       # float32 on the CPU, as torch's _multi_tensor_adam
            lr, (beta1, beta2) = group["lr"], group["betas"]
            scalars = {}                                      # (step_size, bc2_sqrt) per distinct step
            step_sizes, bc2_sqrts = [], []
            for s in [t.item() for t in steps]:
                ss_bc = scalars.get(s)
                if ss_bc is None:
                    ss_bc = scalars[s] = adam_scalars(lr, beta1, beta2, s)
                step_sizes.append(ss_bc[0])
                bc2_sqrts.append(ss_bc[1])
            numels = [p.numel() for p in params]
            if 0 in numels:                                   # nothing to update, but the step still counts
                keep = [i for i, k in enumerate(numels) if k]
                params, grads, exp_avgs, exp_avg_sqs, numels, step_sizes, bc2_sqrts = (
                    [x[i] for i in keep] for x in (params, grads, exp_avgs, exp_avg_sqs, numels, step_sizes, bc2_sqrts))
                if not params:
                    continue
            n = len(params)
            _native.call("wekws_adam_step", _pointers(params), _pointers(grads), _pointers(exp_avgs),
                         _pointers(exp_avg_sqs), (C.c_int64 * n)(*numels), (C.c_double * n)(*step_sizes),
                         (C.c_double * n)(*bc2_sqrts), n, float(beta1), float(beta2), float(group["eps"]),
                         float(group["weight_decay"]), device=params[0].device)
            # the kernel writes through raw pointers: tell autograd and KWSModel's repack check
            torch.autograd.graph.increment_version(params + exp_avgs + exp_avg_sqs)
        return loss


def clip_grad_norm_(parameters, max_norm: float, norm_type: float = 2.0, error_if_nonfinite: bool = False,
                    foreach=None) -> torch.Tensor:
    """torch.nn.utils.clip_grad_norm_ with norm_type 2 in two native launches: returns the total norm as a 0-dim
    float32 tensor on the gradients' device (tensor(0.) on the CPU without gradients) and scales every gradient by
    min(max_norm / (norm + 1e-6), 1) in place, without synchronising.  ``error_if_nonfinite=True`` reads the norm
    back before scaling (two more launches) and raises torch's error.  Refused: another ``norm_type``
    (NotImplementedError), a NaN ``max_norm`` (ValueError), gradients that are not dense contiguous float32 on one
    CUDA device (NotImplementedError).  ``foreach`` selects nothing here."""
    if float(norm_type) != 2.0:
        raise NotImplementedError(f"wekws_b200.clip_grad_norm_: norm_type={norm_type!r} is not supported (2 only)")
    max_norm = float(max_norm)
    if math.isnan(max_norm):
        raise ValueError("wekws_b200.clip_grad_norm_: max_norm is NaN")
    if isinstance(parameters, torch.Tensor):
        parameters = [parameters]
    else:
        is_generator = isinstance(parameters, types.GeneratorType)
        parameters = list(parameters)
        if is_generator and len(parameters) == 0:
            warnings.warn("`parameters` is an empty generator, no gradient clipping will occur.", stacklevel=2)
    grads = [p.grad for p in parameters if p.grad is not None]
    if not grads:
        return torch.tensor(0.0)
    dev = grads[0].device
    for g in grads:
        if g.layout != torch.strided or g.dtype != torch.float32 or g.device != dev or not g.is_contiguous():
            _check_tensor(g, "a gradient", dev)
    if dev.type != "cuda":
        _check_tensor(grads[0], "a gradient")
    grads = [g for g in grads if g.numel()]
    if not grads:
        return torch.zeros((), device=dev)
    n = len(grads)
    ptrs, numels = _pointers(grads), _numels(grads)
    total = sum(numels)
    total_norm = torch.empty((), dtype=torch.float32, device=dev)
    ws = torch.empty(int(_native.lib().wekws_grad_clip_workspace_bytes(n, total)), dtype=torch.uint8, device=dev)
    if error_if_nonfinite:
        _native.call("wekws_grad_clip", ptrs, numels, n, math.nan, total_norm, ws, device=dev)
        if not torch.isfinite(total_norm):
            raise RuntimeError(
                f"The total norm of order {float(norm_type)} for gradients from "
                "`parameters` is non-finite, so it cannot be clipped. To disable "
                "this error and scale the gradients by the non-finite norm anyway, "
                "set `error_if_nonfinite=False`")
    _native.call("wekws_grad_clip", ptrs, numels, n, max_norm, total_norm, ws, device=dev)
    torch.autograd.graph.increment_version(grads)
    return total_norm
