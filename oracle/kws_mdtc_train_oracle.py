"""The MDTC model's training-mode forward in torch, differentiable by autograd (test infrastructure only).

``mdtc_train_logits`` restates wekws/model/kws_model.py with the MDTC backbone and the per-frame linear classifier
in training mode from a ``state_dict``: global CMVN, Linear + ReLU, the preprocessor block and the stacks' blocks
(depthwise dilated causal conv, BatchNorm, pointwise conv, BatchNorm, ReLU, 1x1 conv, BatchNorm, residual, ReLU), the
sum of the stack outputs, the classifier and the activation.  Every BatchNorm is ``F.batch_norm(training=True)``: it
normalises with the batch statistics and updates the running statistics it is given.  Runs in any dtype, on CPU or
CUDA.  Nothing here reads the reference tree.
"""
from typing import Dict, List, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

BLOCK_PARAMS = ["conv1.conv.weight", "conv1.conv.bias", "conv1.bn.weight", "conv1.bn.bias", "conv1.pointwise.weight",
                "conv1.pointwise.bias", "bn1.weight", "bn1.bias", "conv2.weight", "conv2.bias", "bn2.weight", "bn2.bias"]


def blocks(bb: dict) -> List[Tuple[str, int]]:
    """(prefix, dilation) of the preprocessor block and of every stack's blocks, in execution order."""
    out = [("backbone.preprocessor", 1)]
    for s in range(bb["num_stack"]):
        out += [(f"backbone.blocks.{s}.res_blocks.{l}", 2 ** l) for l in range(bb["stack_size"])]
    return out


def param_names(bb: dict) -> List[str]:
    """The model's parameters in named_parameters order (the CMVN and BatchNorm buffers left out)."""
    names = ["preprocessing.out.0.weight", "preprocessing.out.0.bias"]
    for p, _ in blocks(bb):
        names += [f"{p}.{n}" for n in BLOCK_PARAMS]
    return names + ["classifier.linear.weight", "classifier.linear.bias"]


def running_names(bb: dict) -> List[str]:
    """running_mean / running_var of every BatchNorm, block by block (conv1.bn, bn1, bn2)."""
    return [f"{p}.{bn}.{s}" for p, _ in blocks(bb) for bn in ("conv1.bn", "bn1", "bn2")
            for s in ("running_mean", "running_var")]


def mdtc_train_logits(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, running: Dict[str, Tensor],
                      momentum: float = 0.1, eps: float = 1e-5) -> Tuple[Tensor, Tensor]:
    """(logits (B, T, odim), out_cache (B, C, padding)) of the training-mode forward from empty caches.  `running`
    holds the running statistics (running_names) and is updated in place."""
    bb = cfg["backbone"]
    x = feats
    if "global_cmvn.mean" in sd:
        x = x - sd["global_cmvn.mean"]
        if cfg.get("cmvn", {}).get("norm_var", True):
            x = x * sd["global_cmvn.istd"]
    h = F.relu(F.linear(x, sd["preprocessing.out.0.weight"], sd["preprocessing.out.0.bias"])).transpose(1, 2)
    k = bb["kernel_size"]

    def bn(v, p):
        return F.batch_norm(v, running[p + ".running_mean"], running[p + ".running_var"], sd[p + ".weight"],
                            sd[p + ".bias"], training=True, momentum=momentum, eps=eps)

    total, caches = None, []
    for i, (p, d) in enumerate(blocks(bb)):
        padded = F.pad(h, ((k - 1) * d, 0))
        caches.append(padded[:, :, padded.shape[2] - (k - 1) * d:])
        v = F.conv1d(padded, sd[p + ".conv1.conv.weight"], sd[p + ".conv1.conv.bias"], dilation=d, groups=h.shape[1])
        v = F.conv1d(bn(v, p + ".conv1.bn"), sd[p + ".conv1.pointwise.weight"], sd[p + ".conv1.pointwise.bias"])
        v = F.conv1d(F.relu(bn(v, p + ".bn1")), sd[p + ".conv2.weight"], sd[p + ".conv2.bias"])
        h = F.relu(bn(v, p + ".bn2") + h)
        if i > 0 and i % bb["stack_size"] == 0:               # the last block of a stack
            total = h if total is None else total + h
    y = F.linear(total.transpose(1, 2), sd["classifier.linear.weight"], sd["classifier.linear.bias"])
    if cfg.get("activation", {}).get("type") != "identity":
        y = torch.sigmoid(y)
    return y, torch.cat(caches, dim=2)


def mdtc_train_grads(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, upstream: Tensor, dtype=torch.float64,
                     device="cpu") -> Tuple[Tensor, List[Tensor], Dict[str, Tensor], Tensor]:
    """(logits, [d (logits * upstream).sum() / d parameter, in param_names order], the updated running statistics,
    out_cache) computed in ``dtype`` on ``device``."""
    bb = cfg["backbone"]
    names = param_names(bb)
    sdd = {k: v.detach().to(device, dtype).clone() for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    running = {k: sdd[k] for k in running_names(bb)}
    for n in names:
        sdd[n].requires_grad_(True)
    with torch.enable_grad():
        y, cache = mdtc_train_logits(sdd, cfg, feats.detach().to(device, dtype), running)
        (y * upstream.detach().to(device, dtype)).sum().backward()
    return y.detach(), [sdd[n].grad for n in names], {k: v.detach() for k, v in running.items()}, cache.detach()


DIGEST_PROJECTIONS = 3


def digest(t: Tensor) -> Tensor:
    """A float64 fingerprint of a tensor, small enough for a fixture: (max |t|, Sigma |t|, then Sigma r_k t for
    DIGEST_PROJECTIONS fixed N(0, 1) vectors r_k, drawn in float64 on the CPU from generators seeded k = 1, 2, ...).
    Any change of a value shows in the projections at the scale of float64 round-off of the sums."""
    x = t.detach().to("cpu", torch.float64).reshape(-1)
    out = [x.abs().max(), x.abs().sum()]
    for k in range(1, DIGEST_PROJECTIONS + 1):
        r = torch.randn(x.numel(), generator=torch.Generator().manual_seed(k), dtype=torch.float64)
        out.append((r * x).sum())
    return torch.stack(out)


def digest_tolerance(t: Tensor, noise: float) -> Tensor:
    """Per entry of ``digest(t)``: 1e-12 of the sum's own magnitude plus ``noise`` per element (the float64 round-off
    of values that are zero in exact arithmetic, such as the gradient of a bias a BatchNorm cancels)."""
    x = t.detach().to("cpu", torch.float64).reshape(-1)
    tol = [1e-12 * x.abs().max() + noise, 1e-12 * x.abs().sum() + noise * x.numel()]
    for k in range(1, DIGEST_PROJECTIONS + 1):
        r = torch.randn(x.numel(), generator=torch.Generator().manual_seed(k), dtype=torch.float64).abs()
        tol.append(1e-12 * (r * x.abs()).sum() + noise * r.sum())
    return torch.stack(tol)

