"""The FSMN model as the training entry points of csrc/fsmn.cu and csrc/fsmn_grad.cu take it: the parameter order and
the saved activations per frame.  Training runs in training.py."""
from __future__ import annotations

from typing import List


def param_names(num_layers: int) -> List[str]:
    """The parameter order of the native entry points: the FSMN model's ``state_dict`` order without its buffers."""
    names = ["backbone.in_linear1.linear.weight", "backbone.in_linear1.linear.bias",
             "backbone.in_linear2.linear.weight", "backbone.in_linear2.linear.bias"]
    for l in range(num_layers):
        p = f"backbone.fsmn.{l}."
        names += [p + "0.linear.weight", p + "1.conv_left.weight", p + "1.conv_right.weight",
                  p + "2.linear.weight", p + "2.linear.bias"]
    return names + ["backbone.out_linear1.linear.weight", "backbone.out_linear1.linear.bias",
                    "backbone.out_linear2.linear.weight", "backbone.out_linear2.linear.bias"]


def saved_floats_per_frame(bb) -> int:
    """Activations the training forward keeps per frame: in_linear1 and in_linear2 outputs, per layer the projection,
    the memory-block output and the layer output, and the out_linear1 output."""
    return bb.input_affine_dim + bb.linear_dim + bb.fsmn_layers * (2 * bb.proj_dim + bb.linear_dim) + bb.output_affine_dim
