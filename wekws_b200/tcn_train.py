"""The TCN / DS-TCN model as the training entry points of csrc/tcn_train.cu take it: the parameter, BatchNorm and
Dropout order, the saved-activation and launch-count formulas, the limits and the Dropout draw.  Training runs in
training.py."""
from __future__ import annotations

from typing import List, Tuple

import torch.nn as nn

from .frontend import draw_seed

HIDDEN, MAX_K, MAX_LAYERS, MAX_IDIM, MAX_ODIM = (64, 256), 8, 8, 128, 4096


def param_names(num_layers: int, ds: bool) -> List[str]:
    """The parameter order of the native entry points: the TCN / DS-TCN model's ``named_parameters()`` order."""
    names = ["preprocessing.out.0.weight", "preprocessing.out.0.bias"]
    for l in range(num_layers):
        for j in ((0, 1, 3, 4) if ds else (0, 1)):
            names += [f"backbone.network.{l}.cnn.{j}.weight", f"backbone.network.{l}.cnn.{j}.bias"]
    return names + ["classifier.linear.weight", "classifier.linear.bias"]


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


def check_limits(model) -> None:
    """Raises NotImplementedError unless the TCN / DS-TCN `model` is within the training kernels' limits."""
    bb = model.backbone
    if model.hdim not in HIDDEN or not 2 <= bb.kernel_size <= MAX_K or not 1 <= bb.num_layers <= MAX_LAYERS \
            or model.idim > MAX_IDIM or model.odim > MAX_ODIM:
        raise NotImplementedError(f"wekws_b200: {'DS-TCN' if bb.ds else 'TCN'} training supports hidden_dim 64 or 256, "
                                  f"kernel_size 2..{MAX_K}, 1..{MAX_LAYERS} layers, input_dim <= {MAX_IDIM} and "
                                  f"output_dim <= {MAX_ODIM}; got hidden {model.hdim}, kernel {bb.kernel_size}, "
                                  f"{bb.num_layers} layers, input {model.idim}, output {model.odim}")


def draw_dropout(model) -> Tuple[int, List[float]]:
    """(seed, per-block p) of one training forward: one draw from torch's default generator when any p > 0, else
    seed 0."""
    ps = [float(d.p) for d in dropouts(model)]
    return (draw_seed() if any(p > 0 for p in ps) else 0), ps
