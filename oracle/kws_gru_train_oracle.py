"""The GRU model's training-mode forward written out in torch ops, and its parameter gradients by torch's autograd (test
infrastructure only).

``gru_logits`` is wekws/model/kws_model.py with the GRU backbone: global CMVN, the preprocessing Linear + ReLU,
``torch.nn.GRU(hdim, hdim, num_layers, batch_first=True)`` from a zero state with its gates spelled out (PyTorch's
order r, z, n: r = s(W_ir x + b_ir + W_hr h + b_hr), z likewise, n = tanh(W_in x + b_in + r (W_hn h + b_hn)),
h' = (1 - z) n + z h), the linear classifier and the activation.  It runs in any dtype and is differentiable in the
``state_dict`` tensors.  ``gru_grads`` differentiates ``(logits * upstream).sum()``, whose gradient with respect to
the logits is ``upstream``, as ``Executor.train`` differentiates the reference's model.  Nothing here reads the
reference tree.
"""
from typing import Dict, List, Tuple

import torch
from torch import Tensor

from oracle import kws_oracle as O


def param_names(num_layers: int) -> List[str]:
    """The GRU model's parameters in named_parameters order."""
    names = ["preprocessing.out.0.weight", "preprocessing.out.0.bias"]
    for k in range(num_layers):
        names += [f"backbone.{w}_l{k}" for w in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]
    return names + ["classifier.linear.weight", "classifier.linear.bias"]


def gru_logits(sd: Dict[str, Tensor], cfg: dict, feats: Tensor) -> Tuple[Tensor, Tensor]:
    """(logits (B, T, odim), out_cache (L, B, H)) from empty caches, differentiable in the tensors of ``sd``."""
    x = feats
    if "global_cmvn.mean" in sd:
        x = O.global_cmvn(x, sd["global_cmvn.mean"], sd["global_cmvn.istd"], cfg.get("cmvn", {}).get("norm_var", True))
    x = torch.relu(x @ sd["preprocessing.out.0.weight"].t() + sd["preprocessing.out.0.bias"])
    B, T, H = x.shape[0], x.shape[1], x.shape[2]
    last = []
    for k in range(cfg["backbone"]["num_layers"]):
        w_ih, w_hh = sd[f"backbone.weight_ih_l{k}"], sd[f"backbone.weight_hh_l{k}"]
        b_ih, b_hh = sd[f"backbone.bias_ih_l{k}"], sd[f"backbone.bias_hh_l{k}"]
        gi = x @ w_ih.t() + b_ih                                  # (B, T, 3H), every step at once
        h = x.new_zeros(B, H)
        outs = []
        for t in range(T):
            gh = h @ w_hh.t() + b_hh
            r = torch.sigmoid(gi[:, t, :H] + gh[:, :H])
            z = torch.sigmoid(gi[:, t, H:2 * H] + gh[:, H:2 * H])
            n = torch.tanh(gi[:, t, 2 * H:] + r * gh[:, 2 * H:])
            h = (1 - z) * n + z * h
            outs.append(h)
        x = torch.stack(outs, 1) if outs else x.new_zeros(B, 0, H)
        last.append(h)
    y = x @ sd["classifier.linear.weight"].t() + sd["classifier.linear.bias"]
    if cfg.get("activation", {}).get("type", "sigmoid") != "identity":
        y = torch.sigmoid(y)
    return y, torch.stack(last)


def gru_grads(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, upstream: Tensor,
              dtype=torch.float64) -> Tuple[Tensor, List[Tensor]]:
    """(logits, [d (logits * upstream).sum() / d parameter, in param_names order]) computed in ``dtype`` on the CPU."""
    names = param_names(cfg["backbone"]["num_layers"])
    sdd = {k: v.detach().to("cpu", dtype).clone() for k, v in sd.items()}
    for n in names:
        sdd[n].requires_grad_(True)
    with torch.enable_grad():
        y, _ = gru_logits(sdd, cfg, feats.detach().to("cpu", dtype))
        (y * upstream.detach().to("cpu", dtype)).sum().backward()
    return y.detach(), [sdd[n].grad for n in names]


# the golden cases: (input_dim, output_dim, num_layers, activation, global CMVN)
GOLDEN_CASES = {
    "gru": (40, 2, 2, "sigmoid", True),                    # examples/hi_xiaowen/s0/conf/gru.yaml
    "gru_l1_i80": (80, 1, 1, "sigmoid", False),
    "gru_l4_id37": (80, 37, 4, "identity", False),
}


def golden_model(case: str, factory, seed: int = 777):
    """(cfg without the CMVN file, eval-mode model) of a golden case built by `factory` (the reference's or
    wekws_b200's init_model) with synthetic weights."""
    import contextlib
    import io
    import os
    from wekws_b200 import synth
    from wekws_b200.configs import model_config
    idim, odim, layers, act, cmvn = GOLDEN_CASES[case]
    path = synth.write_cmvn_json(idim) if cmvn else None
    try:
        cfg = model_config("gru", input_dim=idim, output_dim=odim, activation=act, cmvn_file=path)
        cfg["backbone"]["num_layers"] = layers
        with contextlib.redirect_stdout(io.StringIO()):
            torch.manual_seed(seed)
            model = factory(cfg)
    finally:
        if path:
            os.unlink(path)
    synth.randomize_(model, seed=seed)
    if "cmvn" in cfg:
        cfg["cmvn"] = dict(norm_var=cfg["cmvn"]["norm_var"])
    return cfg, model.eval()
