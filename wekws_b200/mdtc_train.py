"""The MDTC model as the training entry points of csrc/mdtc_train.cu and csrc/mdtc_head_train.cu take it: the
parameter and BatchNorm order, the saved-activation and launch-count formulas, the limits and, for the ``global`` /
``last`` heads, the Dropout draw.  Training runs in training.py."""
from __future__ import annotations

from typing import List, Tuple

import torch.nn as nn

from .frontend import draw_seed

_BLOCK_PARAMS = ["conv1.conv.weight", "conv1.conv.bias", "conv1.bn.weight", "conv1.bn.bias", "conv1.pointwise.weight",
                 "conv1.pointwise.bias", "bn1.weight", "bn1.bias", "conv2.weight", "conv2.bias", "bn2.weight",
                 "bn2.bias"]
MAX_BLOCKS, MAX_K, MAX_IDIM, MAX_ODIM = 25, 8, 128, 16
HEAD_MAX_ODIM = 4096             # the global / last head's output_dim (Speech Commands v1: 12, v2: 36)
HEAD_WIDTH = 64                  # Linear(hdim, 64) -> ReLU -> Dropout -> Linear(64, odim)
HEAD_DROPOUT_LAYER = 255         # the head's mask: wekws_dropout_mask(seed, B, 1, 64, HEAD_DROPOUT_LAYER, theta)


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


def head_param_names(num_stack: int, stack_size: int) -> List[str]:
    """The parameter order of the head entry points: the MDTC model's ``named_parameters()`` order with the ``global``
    / ``last`` head, classifier.classifier.{0,3} in place of classifier.linear."""
    return param_names(num_stack, stack_size)[:-2] + [f"classifier.classifier.{i}.{n}" for i in (0, 3)
                                                      for n in ("weight", "bias")]


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


def head_saved_floats(num_blocks: int, hdim: int, B: int, T: int) -> int:
    """Floats the grad-mode forward with a head keeps: the backbone's (saved_floats), then per utterance the pooled
    vector and the head's pre-ReLU hidden vector."""
    return saved_floats(num_blocks, hdim, B, T) + B * (hdim + HEAD_WIDTH)


def head_forward_launches(num_blocks: int) -> int:
    """The backbone's forward (its final launch keeps the stack sum and classifies nothing), then the head."""
    return 3 + 3 * num_blocks


def head_backward_launches(num_blocks: int) -> int:
    """The head per utterance; the head's weight sums; per block BN2's gradient statistics, conv2, pointwise and
    depthwise; preprocessing; slice sums."""
    return 4 + 4 * num_blocks


def check_limits(model) -> None:
    """Raises NotImplementedError unless the MDTC `model` is within the training kernels' limits (with a ``global`` /
    ``last`` head: output_dim <= HEAD_MAX_ODIM in place of MAX_ODIM)."""
    bb = model.backbone
    L = 1 + bb.num_stack * bb.stack_size
    max_odim = MAX_ODIM if model.head is None else HEAD_MAX_ODIM
    if model.hdim not in (32, 64) or bb.kernel_size > MAX_K or model.idim > MAX_IDIM or model.odim > max_odim \
            or L > MAX_BLOCKS:
        what = "" if model.head is None else f" with the '{model.head}' head"
        raise NotImplementedError(f"wekws_b200: MDTC training{what} supports hidden_dim 32 or 64, kernel_size <= "
                                  f"{MAX_K}, input_dim <= {MAX_IDIM}, output_dim <= {max_odim} and at most "
                                  f"{MAX_BLOCKS} blocks; got hidden {model.hdim}, kernel {bb.kernel_size}, input "
                                  f"{model.idim}, output {model.odim}, {L} blocks")


def batch_norms(model) -> List[nn.BatchNorm1d]:
    """Every BatchNorm in the order of the native entry points: conv1.bn, bn1, bn2 of each block."""
    bb = model.backbone
    blocks = [bb.preprocessor] + [blk for st in bb.blocks for blk in st.res_blocks]
    return [m for blk in blocks for m in (blk.conv1.bn, blk.bn1, blk.bn2)]


def head_dropout(model) -> nn.Dropout:
    """The ``global`` / ``last`` head's Dropout (classifier.classifier.2)."""
    return model.classifier.classifier[2]


def draw_head_dropout(model) -> Tuple[int, float]:
    """(seed, p) of one training forward with a head: p read from the head's Dropout now, the seed one draw from
    torch's default generator when p > 0, else 0."""
    p = float(head_dropout(model).p)
    return (draw_seed() if p > 0 else 0), p
