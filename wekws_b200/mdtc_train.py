"""The MDTC model as the training entry points of csrc/mdtc_train.cu take it: the parameter and BatchNorm order, the
saved-activation and launch-count formulas and the limits.  Training runs in training.py."""
from __future__ import annotations

from typing import List

import torch.nn as nn

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


def check_limits(model) -> None:
    """Raises NotImplementedError unless the MDTC `model` is within the training kernels' limits."""
    bb = model.backbone
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
