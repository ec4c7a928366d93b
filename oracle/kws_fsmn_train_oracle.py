"""Parameter gradients of the FSMN model by torch's autograd (test infrastructure only).

``fsmn_grads`` differentiates ``kws_oracle``'s FSMN forward (global CMVN, then ``_fsmn``) with the ``state_dict``
tensors requiring grad, as ``Executor.train`` differentiates the reference's model: ``(logits * upstream).sum()`` is
the loss whose gradient with respect to the logits is ``upstream``.  Nothing here reads the reference tree.
"""
from typing import Dict, List, Tuple

import torch
from torch import Tensor

from oracle import kws_oracle as O


def param_names(num_layers: int) -> List[str]:
    """The FSMN model's parameters in state_dict order (its buffers, the CMVN statistics, left out)."""
    names = ["backbone.in_linear1.linear.weight", "backbone.in_linear1.linear.bias",
             "backbone.in_linear2.linear.weight", "backbone.in_linear2.linear.bias"]
    for l in range(num_layers):
        p = f"backbone.fsmn.{l}."
        names += [p + "0.linear.weight", p + "1.conv_left.weight", p + "1.conv_right.weight",
                  p + "2.linear.weight", p + "2.linear.bias"]
    return names + ["backbone.out_linear1.linear.weight", "backbone.out_linear1.linear.bias",
                    "backbone.out_linear2.linear.weight", "backbone.out_linear2.linear.bias"]


def fsmn_logits(sd: Dict[str, Tensor], cfg: dict, feats: Tensor) -> Tensor:
    """The FSMN model's logits from empty caches, differentiable in the tensors of ``sd``."""
    x = feats
    if "global_cmvn.mean" in sd:
        x = O.global_cmvn(x, sd["global_cmvn.mean"], sd["global_cmvn.istd"], cfg.get("cmvn", {}).get("norm_var", True))
    return O._fsmn(x, None, sd, cfg["backbone"])[0]


def fsmn_grads(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, upstream: Tensor,
               dtype=torch.float64) -> Tuple[Tensor, List[Tensor]]:
    """(logits, [d (logits * upstream).sum() / d parameter, in param_names order]) computed in ``dtype`` on the CPU."""
    names = param_names(cfg["backbone"]["num_layers"])
    sdd = {k: v.detach().to("cpu", dtype).clone() for k, v in sd.items()}
    for n in names:
        sdd[n].requires_grad_(True)
    with torch.enable_grad():
        y = fsmn_logits(sdd, cfg, feats.detach().to("cpu", dtype))
        (y * upstream.detach().to("cpu", dtype)).sum().backward()
    return y.detach(), [sdd[n].grad for n in names]
