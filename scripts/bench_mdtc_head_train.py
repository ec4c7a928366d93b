#!/usr/bin/env python
"""Speech-command MDTC training step on the device at the examples/speechcommand_v1/s0/conf/mdtc.yaml sizes (hidden 64,
4 x 4 stacks, 17 blocks, 80-dim MFCC, the `global` head with Dropout 0.5, 11 outputs, criterion ce): B = 100 (the
recipe's batch) and B = 256 one-second clips (T = 98 frames).

Per shape, the p50 of (a) the model's training forward + backward (``y.backward(up)``) and (b) the whole
``Executor.train`` step: forward, ``criterion("ce")``, ``loss.backward()``, ``clip_grad_norm_`` and an Adam step; host
clock ending in a synchronise, after warm-up.  The same two for the same MDTC with the per-frame linear classifier
(one sigmoid output, ``criterion("max_pooling")``) on the device, and for torch's own float32 autograd over the oracle's
training forward with the head (oracle/kws_mdtc_head_train_oracle.py, F.batch_norm in training mode, the same Dropout
masks) on the same card, TF32 off.  Before timing, ours and torch's are compared with the oracle in float64: the largest
error of the logits and of any parameter gradient, relative to that tensor's largest element (ours must be below 1%,
or 8x torch's).  Reports the card and its power limit from the same run.  One JSON line.
      python scripts/bench_mdtc_head_train.py [--steps 20] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import kws_mdtc_head_train_oracle as KH  # noqa: E402
from oracle import kws_mdtc_train_oracle as KM  # noqa: E402
from wekws_b200 import criterion, init_model, mdtc_train, model_config, synth  # noqa: E402
from wekws_b200.frontend import draw_seed  # noqa: E402

SHAPES = [(100, 98), (256, 98)]
ODIM = 11


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


def head_config():
    cfg = model_config("mdtc", output_dim=ODIM)
    cfg["classifier"] = dict(type="global", dropout=0.5)
    return cfg


class Torch(torch.nn.Module):
    """The oracle's training forward with the head as a module with the same parameters and running statistics; each
    call draws its mask's seed from torch's generator, as the device model does."""

    def __init__(self, cfg, sd, p):
        super().__init__()
        self.cfg, self.names, self.p = cfg, KH.param_names(cfg["backbone"]), p
        self.q = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone()) for n in self.names])
        self.running = {k: sd[k].clone() for k in KM.running_names(cfg["backbone"])}

    def forward(self, x):
        mask = KH.head_mask(draw_seed(), x.shape[0], self.p)
        return KH.mdtc_head_train_logits(dict(zip(self.names, self.q)), self.cfg, x, self.running, mask, self.p)[0], None


def torch_ce(type, logits, target, lengths):
    return torch.nn.functional.cross_entropy(logits, target), None


def bench_shape(B, T, dev, steps, warmup):
    cfg = head_config()
    torch.manual_seed(1)
    model = synth.randomize_(init_model(cfg), seed=1)
    p = mdtc_train.head_dropout(model).p
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.to(dev).enable_training(device_dropout=True).train()
    ref = Torch(cfg, {k: v.to(dev) for k, v in sd.items()}, p).to(dev)
    lin_cfg = model_config("mdtc")
    linear = synth.randomize_(init_model(lin_cfg), seed=1).to(dev).enable_training().train()
    gen = torch.Generator().manual_seed(2)
    feats = torch.randn(B, T, cfg["input_dim"], generator=gen).to(dev)
    lens = torch.full((B,), T, device=dev)
    target = torch.randint(0, ODIM, (B,), generator=gen).to(dev)
    kw_target = torch.randint(-1, 1, (B,), generator=gen).to(dev)
    up = torch.randn(B, ODIM, generator=gen).to(dev)
    up_lin = (torch.randn(B, T, 1, generator=gen) * 1e-2).to(dev)

    # both against float64 before anything is timed, with the same mask (the same generator state before each forward)
    torch.manual_seed(3)
    y, _ = model(feats)
    y.backward(up)
    torch.manual_seed(3)
    yr, _ = ref(feats)
    yr.backward(up)
    torch.manual_seed(3)
    mask = KH.head_mask(draw_seed(), B, p)
    y64, g64, _, _ = KH.mdtc_head_train_grads(sd, cfg, feats, up, mask, p, torch.float64, device=dev)
    top = max(float(g.abs().max()) for g in g64)

    def rel(got, want, floor=0.0):
        return float((got.detach().double() - want).abs().max()) / (float(want.abs().max()) + floor)

    ours = max([rel(y, y64)] + [rel(q.grad, g, 1e-6 * top) for q, g in zip(model.parameters(), g64)])
    theirs = max([rel(yr, y64)] + [rel(q.grad, g, 1e-6 * top) for q, g in zip(ref.parameters(), g64)])
    assert ours <= max(1e-2, 8 * theirs), (ours, theirs)
    del g64, y64

    def model_step(m, g):
        def run():
            for q in m.parameters():
                q.grad = None
            out, _ = m(feats)
            out.backward(g)
        return run

    def train_step(m, crit, kind, tgt, opt):
        def run():
            out, _ = m(feats)
            loss, _ = crit(kind, out, tgt, lens)
            opt.zero_grad()
            loss.backward()
            torch.nn.utils.clip_grad_norm_(m.parameters(), 5.0)
            opt.step()
        return run

    res = {"B": B, "T": T, "ours_max_rel_err_vs_f64": ours, "torch_max_rel_err_vs_f64": theirs}
    res["ours_fwd_bwd_ms"] = p50(model_step(model, up), steps, warmup)
    res["linear_fwd_bwd_ms"] = p50(model_step(linear, up_lin), steps, warmup)
    res["torch_fwd_bwd_ms"] = p50(model_step(ref, up), steps, warmup)
    res["ours_train_step_ms"] = p50(train_step(model, criterion, "ce", target,
                                               torch.optim.Adam(model.parameters(), lr=1e-5)), steps, warmup)
    res["linear_train_step_ms"] = p50(train_step(linear, criterion, "max_pooling", kw_target,
                                                 torch.optim.Adam(linear.parameters(), lr=1e-5)), steps, warmup)
    res["torch_train_step_ms"] = p50(train_step(ref, torch_ce, "ce", target,
                                                torch.optim.Adam(ref.parameters(), lr=1e-5)), steps, warmup)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    model_step(model, up)()
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
    out = {"workload": "speech-command mdtc (global head) train step", "card": card(), "torch_tf32": False,
           "shapes": []}
    for B, T in SHAPES:
        out["shapes"].append(bench_shape(B, T, dev, args.steps, args.warmup))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
