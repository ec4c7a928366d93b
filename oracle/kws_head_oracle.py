"""CPU oracle of the utterance-level classifier heads (reference wekws/model/classifier.py:19-40 behind
kws_model.py:175-195): the backbone of kws_oracle, then GlobalClassifier (mean over all T frames of the call,
zero-padded frames included) or LastClassifier (frame T-1) around Linear(H, 64) -> ReLU -> Dropout (eval: identity)
-> Linear(64, odim); activation Identity.  Models without a head go to kws_oracle.kws_forward unchanged."""
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F
from torch import Tensor

from . import kws_oracle as O


@torch.no_grad()
def kws_forward(sd: Dict[str, Tensor], cfg: dict, feats: Tensor,
                cache: Optional[Tensor] = None) -> Tuple[Tensor, Tensor]:
    """KWSModel.forward with the head of cfg['classifier'] when the state dict carries one: logits (B, odim)."""
    if "classifier.classifier.0.weight" not in sd:
        return O.kws_forward(sd, cfg, feats, cache)
    if cache is not None and cache.numel() == 0:
        cache = None
    x = feats
    if "global_cmvn.mean" in sd:
        x = O.global_cmvn(x, sd["global_cmvn.mean"], sd["global_cmvn.istd"], cfg.get("cmvn", {}).get("norm_var", True))
    bb = cfg["backbone"]
    x = F.relu(F.linear(x, sd["preprocessing.out.0.weight"], sd["preprocessing.out.0.bias"]))
    if bb["type"] == "mdtc":
        x, new_cache = O._mdtc(x, cache, sd, bb)
    elif bb["type"] == "tcn":
        x, new_cache = O._tcn(x, cache, sd, bb)
    else:
        raise ValueError("head oracle: unsupported backbone " + str(bb["type"]))
    x = torch.mean(x, dim=1) if cfg["classifier"]["type"] == "global" else x[:, -1, :]
    x = F.relu(F.linear(x, sd["classifier.classifier.0.weight"], sd["classifier.classifier.0.bias"]))
    x = F.linear(x, sd["classifier.classifier.3.weight"], sd["classifier.classifier.3.bias"])
    return x, new_cache
