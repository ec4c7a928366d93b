#!/usr/bin/env python
"""FSMN training step on the device at the fsmn_ctc.yaml sizes (400 / 140 / 250 / 128, L = 4, lo = 10, ro = 2,
V = 2599): B = 256 utterances of T = 200 frames, lengths uniform in [100, 200], labels of up to 30 tokens.

Reports the p50 of (a) the model's training forward + backward (``y.backward(up)``) and (b) the whole step with
``criterion("ctc")`` (forward, loss, ``loss.backward()``), host clock ending in a synchronise, after warm-up; the same
two for torch's own float32 autograd over the oracle's FSMN forward on the same card; per-kernel times from
torch.profiler in a separate run; FLOPs from shapes and the share of the FP32 rate; the card and its power limit.
One JSON line.
      python scripts/bench_fsmn_train.py [--steps 20] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import kws_criterion_oracle as K  # noqa: E402
from oracle import kws_fsmn_train_oracle as KF  # noqa: E402
from wekws_b200 import criterion, init_model, model_config  # noqa: E402

B, T, V, MAXLAB = 256, 200, 2599, 30
FP32_TFLOPS = 67.0               # H100 SXM data sheet, non-tensor FP32


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


def flops(bb, frames):
    """Multiply-adds of the forward per frame x 2 FLOPs; the backward is twice the forward's GEMMs (dX and dW) and
    twice its memory-block taps."""
    P, D, L = bb.proj_dim, bb.linear_dim, bb.fsmn_layers
    gemm = bb.input_dim * bb.input_affine_dim + bb.input_affine_dim * D + L * (2 * D * P) + D * bb.output_affine_dim \
        + bb.output_affine_dim * bb.output_dim
    taps = L * P * (bb.lorder + bb.rorder)
    fwd = 2 * frames * (gemm + taps)
    return fwd, 2 * fwd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    cfg = model_config("fsmn", input_dim=400, output_dim=V)
    model = init_model(cfg).to(dev).train()
    gen = torch.Generator().manual_seed(1)
    feats = torch.randn(B, T, 400, generator=gen).to(dev)
    lens = torch.randint(100, T + 1, (B,), generator=gen)
    tl = torch.randint(1, MAXLAB + 1, (B,), generator=gen)
    labels = torch.randint(1, V, (B, MAXLAB), generator=gen)
    lens, tl, labels = lens.to(dev), tl.to(dev), labels.to(dev)
    up = (torch.randn(B, T, V, generator=gen) * 1e-3).to(dev)
    params = list(model.parameters())

    def model_step(m, f):
        def run():
            for p in params_of[m]:
                p.grad = None
            y, _ = m(f)
            y.backward(up)
        return run

    def full_step(m, crit):
        def run():
            for p in params_of[m]:
                p.grad = None
            y, _ = m(feats)
            loss, _ = crit("ctc", y, labels, lens, tl)
            loss.backward()
        return run

    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    names = KF.param_names(4)

    class Torch(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.p = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone()) for n in names])

        def forward(self, x):
            return KF.fsmn_logits(dict(zip(names, self.p)), cfg, x), None

    ref = Torch().to(dev)
    params_of = {model: params, ref: list(ref.parameters())}

    res = {"workload": "fsmn_ctc train step", "B": B, "T": T, "V": V, "card": card()}
    res["ours_model_fwd_bwd_ms"] = p50(model_step(model, feats), args.steps, args.warmup)
    res["ours_step_ctc_ms"] = p50(full_step(model, criterion), args.steps, args.warmup)
    res["torch_model_fwd_bwd_ms"] = p50(model_step(ref, feats), args.steps, args.warmup)
    res["torch_step_ctc_ms"] = p50(full_step(ref, K.criterion), args.steps, args.warmup)
    fwd, bwd = flops(model.backbone, B * T)
    res["tflop_fwd_bwd"] = (fwd + bwd) / 1e12
    res["ours_fp32_share"] = (fwd + bwd) / (res["ours_model_fwd_bwd_ms"] * 1e-3) / (FP32_TFLOPS * 1e12)
    res["torch_fp32_share"] = (fwd + bwd) / (res["torch_model_fwd_bwd_ms"] * 1e-3) / (FP32_TFLOPS * 1e12)
    res["peak_mem_gb_ours_step"] = None
    torch.cuda.reset_peak_memory_stats()
    full_step(model, criterion)()
    torch.cuda.synchronize()
    res["peak_mem_gb_ours_step"] = torch.cuda.max_memory_allocated() / 1e9

    # per-kernel times of our model step, separate run
    from torch.profiler import ProfilerActivity, profile
    run = model_step(model, feats)
    run()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            run()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0) > 0:
            t = getattr(e, "self_device_time_total", None)
            if t is None:
                t = e.self_cuda_time_total
            if t > 0:
                kern[e.key] = {"ms_per_step": t / 1e3 / 3, "calls_per_step": e.count / 3}
    res["kernels"] = dict(sorted(kern.items(), key=lambda kv: -kv[1]["ms_per_step"])[:12])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
