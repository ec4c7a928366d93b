"""The GRU model as the training entry points of csrc/gru.cu and csrc/gru_train.cu take it: the parameter order, the
activations the training forward keeps per frame, and the kernels' limits.  Training runs in training.py."""
from __future__ import annotations

from typing import List

import torch.nn as nn

HIDDEN = 128                 # the fused kernels' hidden width (one thread per gate row)
MAX_LAYERS = 4
MAX_INPUT_DIM = 128


def param_names(num_layers: int) -> List[str]:
    """The parameter order of the native entry points: the model's ``named_parameters`` order."""
    names = ["preprocessing.out.0.weight", "preprocessing.out.0.bias"]
    for k in range(num_layers):
        names += [f"backbone.{w}_l{k}" for w in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return names + ["classifier.linear.weight", "classifier.linear.bias"]


def saved_floats_per_frame(num_layers: int, hidden: int = HIDDEN) -> int:
    """Activations the training forward keeps per frame: the layer-0 input, then per layer h_t, r, z, n and
    W_hn h_{t-1} + b_hn."""
    return (1 + 5 * num_layers) * hidden


def check_limits(model) -> None:
    """Raises NotImplementedError for a GRU model outside what the training kernels accept."""
    bb = model.backbone
    if bb.dropout > 0:
        raise NotImplementedError(f"wekws_b200: GRU training does not implement nn.GRU's inter-layer Dropout "
                                  f"(dropout={bb.dropout}); build the GRU with dropout=0")
    if bb.hidden_size != HIDDEN or not 1 <= bb.num_layers <= MAX_LAYERS or not 1 <= model.idim <= MAX_INPUT_DIM:
        raise NotImplementedError(f"wekws_b200: GRU training supports hidden_dim {HIDDEN}, 1..{MAX_LAYERS} layers and "
                                  f"input_dim 1..{MAX_INPUT_DIM} (output_dim is not limited); got hidden_dim "
                                  f"{bb.hidden_size}, {bb.num_layers} layers, input_dim {model.idim}")
    if not isinstance(model.activation, (nn.Sigmoid, nn.Identity)):
        raise NotImplementedError("wekws_b200: GRU training needs the Sigmoid or Identity activation")
