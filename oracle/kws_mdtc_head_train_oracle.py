"""The speech-command MDTC model's training-mode forward in torch, differentiable by autograd (test infrastructure
only).

``mdtc_head_train_logits`` restates wekws/model/kws_model.py with the MDTC backbone and the ``global`` / ``last`` head
(wekws/model/classifier.py GlobalClassifier / LastClassifier around Linear(C, 64), ReLU, Dropout, Linear(64, odim)) in
training mode from a ``state_dict``.  The backbone is kws_mdtc_train_oracle's, up to the stack sum: its per-frame
classifier is given the C x C identity and zero bias with the identity activation, which returns the stack sum exactly
(one product with 1 and C - 1 products with 0 per element, in the forward and in the backward).  The head pools (the
mean over all T frames, padding included, as torch.mean; or frame T - 1), and its Dropout multiplies by the given
boolean mask (B, 64) times the scale 1 / (1 - p) (``1.0f / (float)(1 - p)`` in float32, torch's scale).  ``head_mask``
regenerates the device mask in numpy from the seed.  Runs in any dtype, on CPU or CUDA.  Nothing here reads the
reference tree.
"""
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import kws_mdtc_train_oracle as KM
from oracle import kws_tcn_train_oracle as KT

HEAD_WIDTH = 64
DROPOUT_LAYER = 255        # Philox counter word 3 = 1 + 255 = 256: apart from the dither (0) and the TCN blocks (1..8)
HEAD_PARAMS = [f"classifier.classifier.{i}.{n}" for i in (0, 3) for n in ("weight", "bias")]


def param_names(bb: dict) -> List[str]:
    """The model's parameters in named_parameters order: the MDTC backbone's, then the head's."""
    return KM.param_names(bb)[:-2] + HEAD_PARAMS


def head_mask(seed: int, B: int, p: float) -> np.ndarray:
    """(B, 64) bool, True where the head's Dropout keeps element (b, j): component j % 4 of Philox4x32-10(counter =
    (j // 4, 0, b, 256), key = (seed lo, seed hi)), kept iff (word >> 8) >= ceil(p 2^24)."""
    return KT.dropout_mask(seed, B, 1, HEAD_WIDTH, DROPOUT_LAYER, p)[:, 0, :]


def stack_sum(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, running: Dict[str, Tensor]) -> Tuple[Tensor, Tensor]:
    """(the MDTC backbone's stack sum (B, T, C), out_cache (B, C, padding)) of the training-mode forward; `running` is
    updated in place."""
    C = sd["preprocessing.out.0.bias"].shape[0]
    ref = sd["preprocessing.out.0.bias"]
    eye = dict(sd)
    eye["classifier.linear.weight"] = torch.eye(C, dtype=ref.dtype, device=ref.device)
    eye["classifier.linear.bias"] = torch.zeros(C, dtype=ref.dtype, device=ref.device)
    return KM.mdtc_train_logits(eye, dict(cfg, activation=dict(type="identity")), feats, running)


def mdtc_head_train_logits(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, running: Dict[str, Tensor],
                           mask: Optional[Tensor], p: float) -> Tuple[Tensor, Tensor]:
    """(logits (B, odim), out_cache (B, C, padding)) of the training-mode forward from empty caches.  `mask`: (B, 64)
    bool (None: no Dropout); `running` is updated in place."""
    s, cache = stack_sum(sd, cfg, feats, running)
    pool = s.mean(dim=1) if cfg["classifier"]["type"] == "global" else s[:, -1, :]
    h = F.relu(F.linear(pool, sd["classifier.classifier.0.weight"], sd["classifier.classifier.0.bias"]))
    if mask is not None:                             # p = 1 drops every element: no scale is needed (nor finite)
        m = torch.as_tensor(mask).to(h.device)
        sc = KT.scale(p, h.dtype) if p < 1 else torch.zeros((), dtype=h.dtype)
        h = h * torch.where(m, sc.to(h.device), torch.zeros((), dtype=h.dtype, device=h.device))
    return F.linear(h, sd["classifier.classifier.3.weight"], sd["classifier.classifier.3.bias"]), cache


def mdtc_head_train_grads(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, upstream: Tensor, mask, p: float,
                          dtype=torch.float64, device="cpu"):
    """(logits, [d (logits * upstream).sum() / d parameter, in param_names order], the updated running statistics,
    out_cache) computed in ``dtype`` on ``device``."""
    bb = cfg["backbone"]
    names = param_names(bb)
    sdd = {k: v.detach().to(device, dtype).clone() for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    running = {k: sdd[k] for k in KM.running_names(bb)}
    for n in names:
        sdd[n].requires_grad_(True)
    with torch.enable_grad():
        y, cache = mdtc_head_train_logits(sdd, cfg, feats.detach().to(device, dtype), running, mask, p)
        (y * upstream.detach().to(device, dtype)).sum().backward()
    return y.detach(), [sdd[n].grad for n in names], {k: v.detach() for k, v in running.items()}, cache.detach()
