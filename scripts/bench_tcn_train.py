#!/usr/bin/env python
"""Times one training step's model side (forward + backward of (logits * up).sum()) of the TCN / DS-TCN models on the
device against torch's FP32 autograd of the same model (kws_tcn_train_oracle, same Dropout masks), with TF32 off and
with torch's defaults, at the recipes' batch_size B = 256 and T = 200 frames.  Prints the card and its power limit.
    python scripts/bench_tcn_train.py [--B 256] [--T 200] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import kws_tcn_train_oracle as KT  # noqa: E402
from wekws_b200 import init_model, model_config, synth, tcn_train  # noqa: E402
from wekws_b200.frontend import draw_seed  # noqa: E402

CASES = [("tcn 64", "tcn", {}), ("ds_tcn 64", "ds_tcn", dict(hidden=64)), ("ds_tcn 256", "ds_tcn", {}),
         ("ds_tcn 256, odim 2599", "ds_tcn", dict(activation="identity", output_dim=2599, input_dim=80))]


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--T", type=int, default=200)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    B, T = args.B, args.T
    for label, name, kw in CASES:
        kw = dict(kw)
        hidden = kw.pop("hidden", None)
        cfg = model_config(name, **kw)
        if hidden:
            cfg["hidden_dim"] = hidden
        torch.manual_seed(0)
        model = synth.randomize_(init_model(cfg), seed=0).to(dev).enable_training(device_dropout=True).train()
        sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
        ps = [d.p for d in tcn_train.dropouts(model)]
        x = torch.randn(B, T, cfg["input_dim"], device=dev)
        up = torch.randn(B, T, cfg["output_dim"], device=dev)

        def ours():
            y, _ = model(x)
            (y * up).sum().backward()

        masks = [torch.from_numpy(m).to(dev) for m in KT.dropout_masks(draw_seed(), B, T, cfg["hidden_dim"], ps)]
        names = KT.param_names(cfg["backbone"])
        sdt = {k: (v.clone().requires_grad_(True) if k in names else v.clone()) for k, v in sd.items()
               if not k.endswith("num_batches_tracked")}
        running = {k: sdt[k] for k in KT.running_names(cfg["backbone"])}

        def torch_step():
            y, _ = KT.tcn_train_logits(sdt, cfg, x, running, masks, ps)
            (y * up).sum().backward()

        t_ours = timed(ours, args.iters)
        tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        t_fp32 = timed(torch_step, args.iters)
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        t_def = timed(torch_step, args.iters)
        print(json.dumps(dict(model=label, B=B, T=T, device_ms=round(t_ours, 3), torch_fp32_ms=round(t_fp32, 3),
                              torch_default_ms=round(t_def, 3), card=card)))


if __name__ == "__main__":
    main()
