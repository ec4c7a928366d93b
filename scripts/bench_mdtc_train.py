#!/usr/bin/env python
"""MDTC training step on the device at the mdtc.yaml sizes (hidden 64, 4 x 4 stacks, 17 blocks, 80-dim features,
one sigmoid output): B = 100 utterances of T = 200 and T = 1000 frames, lengths uniform in [T / 2, T]; and mdtc_small
(hidden 32, 3 x 4) at T = 200.

Per shape, the p50 of (a) the model's training forward + backward (``y.backward(up)``) and (b) the whole
``Executor.train`` step: forward, ``criterion("max_pooling")``, ``loss.backward()``, ``clip_grad_norm_`` and an Adam
step; host clock ending in a synchronise, after warm-up.  The same two for torch's own float32 autograd over the
oracle's training forward (oracle/kws_mdtc_train_oracle.py, F.batch_norm in training mode) on the same card, TF32
off.  Before timing, both are compared with the oracle in float64: the largest error of the logits and of any
parameter gradient, relative to that tensor's largest element, is reported for each (ours must be below 1%, or 8x torch's).  Reports
the card and its power limit from the same run.  One JSON line.
      python scripts/bench_mdtc_train.py [--steps 20] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import kws_mdtc_train_oracle as KM  # noqa: E402
from wekws_b200 import criterion, init_model, model_config, synth  # noqa: E402

SHAPES = [("mdtc", 100, 200), ("mdtc", 100, 1000), ("mdtc_small", 100, 200)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def p50(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    ts.sort()
    return ts[len(ts) // 2] * 1e3


def torch_max_pooling(type, logits, target, lengths):
    """loss.py max_pooling_loss (one keyword, min_duration 0) in vectorised torch ops on the logits' device: the
    baseline step's criterion.  Returns (loss, None)."""
    B, T, _ = logits.shape
    mask = torch.arange(T, device=logits.device)[None, :] >= lengths[:, None]
    p = logits[:, :, 0].masked_fill(mask, 0.0).clamp(1e-8, 1.0 - 1e-8)
    top = p.max(dim=1).values
    loss = torch.where(target == 0, -torch.log(top), -torch.log(1.0 - top))
    return loss.sum() / B, None


class Torch(torch.nn.Module):
    """The oracle's training forward as a module with the same parameters and running statistics."""

    def __init__(self, cfg, sd):
        super().__init__()
        self.cfg, self.names = cfg, KM.param_names(cfg["backbone"])
        self.p = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone()) for n in self.names])
        self.running = {k: sd[k].clone() for k in KM.running_names(cfg["backbone"])}

    def forward(self, x):
        return KM.mdtc_train_logits(dict(zip(self.names, self.p)), self.cfg, x, self.running)[0], None


def bench_shape(name, B, T, dev, steps, warmup):
    cfg = model_config(name)
    model = synth.randomize_(init_model(cfg), seed=1)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.to(dev).enable_training().train()
    ref = Torch(cfg, {k: v.to(dev) for k, v in sd.items()}).to(dev)
    gen = torch.Generator().manual_seed(2)
    feats = torch.randn(B, T, cfg["input_dim"], generator=gen).to(dev)
    lens = torch.randint(T // 2, T + 1, (B,), generator=gen).to(dev)
    target = torch.randint(-1, 1, (B,), generator=gen).to(dev)
    up = (torch.randn(B, T, 1, generator=gen) * 1e-2).to(dev)

    # both against float64 before anything is timed: the largest error of the logits and of each gradient, relative to
    # that tensor's largest float64 element (a model-wide floor of 1e-6 of the largest gradient for the biases a
    # BatchNorm cancels, whose gradients are zero up to round-off)
    y, _ = model(feats)
    y.backward(up)
    yr, _ = ref(feats)
    yr.backward(up)
    y64, g64, _, _ = KM.mdtc_train_grads(sd, cfg, feats, up, torch.float64, device=dev)
    top = max(float(g.abs().max()) for g in g64)

    def rel(got, want, floor=0.0):
        return float((got.detach().double() - want).abs().max()) / (float(want.abs().max()) + floor)

    ours = max([rel(y, y64)] + [rel(q.grad, g, 1e-6 * top) for q, g in zip(model.parameters(), g64)])
    theirs = max([rel(yr, y64)] + [rel(p.grad, g, 1e-6 * top) for p, g in zip(ref.parameters(), g64)])
    assert ours <= max(1e-2, 8 * theirs), (ours, theirs)
    del g64, y64

    def model_step(m):
        def run():
            for p in m.parameters():
                p.grad = None
            out, _ = m(feats)
            out.backward(up)
        return run

    def train_step(m, crit, opt):
        def run():
            out, _ = m(feats)
            loss, _ = crit("max_pooling", out, target, lens)
            opt.zero_grad()
            loss.backward()
            torch.nn.utils.clip_grad_norm_(m.parameters(), 5.0)
            opt.step()
        return run

    res = {"model": name, "B": B, "T": T, "ours_max_rel_err_vs_f64": ours, "torch_max_rel_err_vs_f64": theirs}
    res["ours_fwd_bwd_ms"] = p50(model_step(model), steps, warmup)
    res["torch_fwd_bwd_ms"] = p50(model_step(ref), steps, warmup)
    res["ours_train_step_ms"] = p50(train_step(model, criterion, torch.optim.Adam(model.parameters(), lr=1e-5)),
                                    steps, warmup)
    res["torch_train_step_ms"] = p50(train_step(ref, torch_max_pooling, torch.optim.Adam(ref.parameters(), lr=1e-5)),
                                     steps, warmup)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    model_step(model)()
    torch.cuda.synchronize()
    res["ours_peak_mem_gb"] = torch.cuda.max_memory_allocated(dev) / 1e9
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False          # torch in FP32, as the device kernels
    torch.backends.cuda.matmul.allow_tf32 = False
    out = {"workload": "mdtc train step", "card": card(), "torch_tf32": False, "shapes": []}
    for name, B, T in SHAPES:
        out["shapes"].append(bench_shape(name, B, T, dev, args.steps, args.warmup))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
