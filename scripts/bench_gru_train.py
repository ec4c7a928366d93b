#!/usr/bin/env python
"""Times one training step's model side (forward + backward of (logits * up).sum()) of the GRU model of
examples/hi_xiaowen/s0/conf/gru.yaml (input_dim 40, output_dim 2, global CMVN, 2 layers) on the device against torch's
training step of the same model on the same GPU (CMVN, nn.Linear + ReLU, cuDNN nn.GRU, nn.Linear, Sigmoid), with TF32
off and with torch's defaults, at the recipe's batch_size B = 256 and T = 200 and 1000 frames.  Prints the card and
its power limit.
    python scripts/bench_gru_train.py [--B 256] [--T 200 1000] [--iters 10]"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import kws_gru_train_oracle as KG  # noqa: E402
from wekws_b200 import init_model  # noqa: E402


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


class TorchGru(torch.nn.Module):
    """The same model in torch modules: the GRU runs on cuDNN."""

    def __init__(self, sd, idim, odim, layers):
        super().__init__()
        self.register_buffer("mean", sd["global_cmvn.mean"].clone())
        self.register_buffer("istd", sd["global_cmvn.istd"].clone())
        self.pre = torch.nn.Linear(idim, 128)
        self.gru = torch.nn.GRU(128, 128, num_layers=layers, batch_first=True)
        self.cls = torch.nn.Linear(128, odim)
        with torch.no_grad():
            self.pre.weight.copy_(sd["preprocessing.out.0.weight"])
            self.pre.bias.copy_(sd["preprocessing.out.0.bias"])
            for n, p in self.gru.named_parameters():
                p.copy_(sd["backbone." + n])
            self.cls.weight.copy_(sd["classifier.linear.weight"])
            self.cls.bias.copy_(sd["classifier.linear.bias"])

    def forward(self, x):
        x = torch.relu(self.pre((x - self.mean) * self.istd))
        return torch.sigmoid(self.cls(self.gru(x)[0]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--T", type=int, nargs="+", default=[200, 1000])
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    cfg, model = KG.golden_model("gru", init_model, seed=0)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    model = model.to(dev).enable_training(bptt=True).train()
    ref = TorchGru(sd, cfg["input_dim"], cfg["output_dim"], cfg["backbone"]["num_layers"]).to(dev).train()
    B = args.B
    for T in args.T:
        x = torch.randn(B, T, cfg["input_dim"], device=dev) * 3 + 15
        up = torch.randn(B, T, cfg["output_dim"], device=dev)

        def ours():
            y, _ = model(x)
            (y * up).sum().backward()

        def torch_step():
            (ref(x) * up).sum().backward()

        t_ours = timed(ours, args.iters)
        tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        t_fp32 = timed(torch_step, args.iters)
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
        t_def = timed(torch_step, args.iters)
        print(json.dumps(dict(model="gru", B=B, T=T, device_ms=round(t_ours, 3), torch_fp32_ms=round(t_fp32, 3),
                              torch_default_ms=round(t_def, 3), card=card)))


if __name__ == "__main__":
    main()
