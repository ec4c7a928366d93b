"""The TCN / DS-TCN model's training-mode forward in torch, differentiable by autograd (test infrastructure only).

``tcn_train_logits`` restates wekws/model/kws_model.py with the TCN backbone (wekws/model/tcn.py, CnnBlock or
DsCnnBlock) and the per-frame linear classifier in training mode from a ``state_dict``: global CMVN, Linear + ReLU,
per block the causal dilated conv, BatchNorm, ReLU [, 1x1 conv, BatchNorm, ReLU], Dropout, residual; the classifier
and the activation.  Every BatchNorm is ``F.batch_norm(training=True)``.  Dropout multiplies by the given boolean masks
(B, T, C) times the scale 1 / (1 - p) (``1.0f / (float)(1 - p)`` in float32, torch's scale).  ``dropout_masks``
regenerates the device masks in numpy from the seed.  Runs in any dtype, on CPU or CUDA.  Nothing here reads the
reference tree.
"""
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from oracle.kws_train_oracle import philox4x32_10


def param_names(bb: dict) -> List[str]:
    names = ["preprocessing.out.0.weight", "preprocessing.out.0.bias"]
    for l in range(bb["num_layers"]):
        for j in ((0, 1, 3, 4) if bb.get("ds", False) else (0, 1)):
            names += [f"backbone.network.{l}.cnn.{j}.weight", f"backbone.network.{l}.cnn.{j}.bias"]
    return names + ["classifier.linear.weight", "classifier.linear.bias"]


def running_names(bb: dict) -> List[str]:
    return [f"backbone.network.{l}.cnn.{j}.{s}" for l in range(bb["num_layers"])
            for j in ((1, 4) if bb.get("ds", False) else (1,)) for s in ("running_mean", "running_var")]


def theta(p: float) -> int:
    """ceil(p 2^24) in double: the keep threshold on the top 24 bits of a Philox word."""
    return int(np.ceil(p * 2.0 ** 24))


def dropout_mask(seed: int, B: int, T: int, C: int, layer: int, p: float) -> np.ndarray:
    """(B, T, C) bool, True where block `layer` keeps the element: component c % 4 of Philox4x32-10(counter =
    (c // 4, t, b, 1 + layer), key = (seed lo, seed hi)), kept iff (word >> 8) >= theta(p)."""
    q, t, b = np.meshgrid(np.arange((C + 3) // 4), np.arange(T), np.arange(B), indexing="ij")
    ctr = np.stack([q, t, b, np.full_like(q, 1 + layer)], axis=-1).astype(np.uint32)
    w = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32))                        # (q, t, b, 4)
    w = w.transpose(2, 1, 0, 3).reshape(B, T, -1)[:, :, :C]
    return (w >> np.uint32(8)) >= np.uint32(theta(p))


def dropout_masks(seed: int, B: int, T: int, C: int, ps) -> List[np.ndarray]:
    return [dropout_mask(seed, B, T, C, l, p) for l, p in enumerate(ps)]


def scale(p: float, dtype) -> Tensor:
    if dtype == torch.float32:
        return torch.tensor(np.float32(1.0) / np.float32(1.0 - p))
    return torch.tensor(1.0 / (1.0 - p), dtype=dtype)


def tcn_train_logits(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, running: Dict[str, Tensor],
                     masks: Optional[List[Tensor]], ps, momentum: float = 0.1, eps: float = 1e-5) -> Tuple[Tensor, Tensor]:
    """(logits (B, T, odim), out_cache (B, C, padding)) of the training-mode forward from empty caches.  `masks`: per
    block (B, T, C) bool (None: no Dropout); `running` is updated in place."""
    bb = cfg["backbone"]
    ds, k = bb.get("ds", False), bb.get("kernel_size", 8)
    x = feats
    if "global_cmvn.mean" in sd:
        x = x - sd["global_cmvn.mean"]
        if cfg.get("cmvn", {}).get("norm_var", True):
            x = x * sd["global_cmvn.istd"]
    h = F.relu(F.linear(x, sd["preprocessing.out.0.weight"], sd["preprocessing.out.0.bias"])).transpose(1, 2)

    def bn(v, p):
        return F.batch_norm(v, running[p + ".running_mean"], running[p + ".running_var"], sd[p + ".weight"],
                            sd[p + ".bias"], training=True, momentum=momentum, eps=eps)

    caches = []
    for l in range(bb["num_layers"]):
        d, p = 2 ** l, f"backbone.network.{l}.cnn"
        padded = F.pad(h, ((k - 1) * d, 0))
        caches.append(padded[:, :, padded.shape[2] - (k - 1) * d:])
        v = F.conv1d(padded, sd[p + ".0.weight"], sd[p + ".0.bias"], dilation=d, groups=h.shape[1] if ds else 1)
        v = F.relu(bn(v, p + ".1"))
        if ds:
            v = F.relu(bn(F.conv1d(v, sd[p + ".3.weight"], sd[p + ".3.bias"]), p + ".4"))
        if masks is not None:
            m = masks[l].to(v.device).transpose(1, 2)
            v = v * torch.where(m, scale(ps[l], v.dtype).to(v.device), torch.zeros((), dtype=v.dtype, device=v.device))
        h = v + h
    y = F.linear(h.transpose(1, 2), sd["classifier.linear.weight"], sd["classifier.linear.bias"])
    if cfg.get("activation", {}).get("type") != "identity":
        y = torch.sigmoid(y)
    return y, torch.cat(caches, dim=2)


def tcn_train_grads(sd: Dict[str, Tensor], cfg: dict, feats: Tensor, upstream: Tensor, masks, ps,
                    dtype=torch.float64, device="cpu"):
    """(logits, [d (logits * upstream).sum() / d parameter, in param_names order], the updated running statistics,
    out_cache) computed in ``dtype`` on ``device``."""
    bb = cfg["backbone"]
    names = param_names(bb)
    sdd = {k: v.detach().to(device, dtype).clone() for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    running = {k: sdd[k] for k in running_names(bb)}
    for n in names:
        sdd[n].requires_grad_(True)
    masks = None if masks is None else [torch.as_tensor(m) for m in masks]
    with torch.enable_grad():
        y, cache = tcn_train_logits(sdd, cfg, feats.detach().to(device, dtype), running, masks, ps)
        (y * upstream.detach().to(device, dtype)).sum().backward()
    return y.detach(), [sdd[n].grad for n in names], {k: v.detach() for k, v in running.items()}, cache.detach()


# The golden cases (oracle/make_tcn_train_golden.py, tests/test_tcn_train_host.py): name -> (config name,
# model_config kwargs, hidden_dim override, global CMVN with norm_var, every block's Dropout p or None for the config's)
GOLDEN_CASES = {
    "tcn": ("tcn", dict(), None, None, None),
    "ds_tcn": ("ds_tcn", dict(), None, None, None),
    "ds_tcn64_cmvn": ("ds_tcn", dict(input_dim=40, output_dim=2), 64, True, None),
    "ds_tcn_ctc": ("ds_tcn", dict(activation="identity", output_dim=37, input_dim=40), None, None, None),
    "ds_tcn64_p0": ("ds_tcn", dict(), 64, None, 0.0),
}


def golden_config(case: str):
    """(model config, cleanup) of a golden case; the config may name a temporary CMVN file that cleanup removes."""
    import os
    from wekws_b200 import synth
    from wekws_b200.configs import model_config
    name, kw, hidden, cmvn, _ = GOLDEN_CASES[case]
    path = synth.write_cmvn_json(kw.get("input_dim", 80)) if cmvn is not None else None
    cfg = model_config(name, cmvn_file=path, norm_var=bool(cmvn), **kw)
    if hidden is not None:
        cfg["hidden_dim"] = hidden
    return cfg, (lambda: os.unlink(path)) if path else (lambda: None)


def golden_model(case: str, factory, seed: int = 777):
    """(cfg without the CMVN file, model) of a golden case built by `factory` (the reference's or wekws_b200's
    init_model) with synthetic weights, every block's Dropout p set as the case says."""
    import contextlib
    import io
    from wekws_b200 import synth
    cfg, cleanup = golden_config(case)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            torch.manual_seed(seed)
            model = factory(cfg)
    finally:
        cleanup()
    synth.randomize_(model, seed=seed)
    p = GOLDEN_CASES[case][4]
    if p is not None:
        for blk in model.backbone.network:
            blk.cnn[-1].p = p
    if "cmvn" in cfg:
        cfg["cmvn"] = dict(norm_var=cfg["cmvn"]["norm_var"])
    return cfg, model.eval()


def block_dropouts(model) -> List[torch.nn.Module]:
    return [blk.cnn[-1] for blk in model.backbone.network]
