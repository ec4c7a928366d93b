#!/usr/bin/env python
"""Times one training step's criterion, forward + backward (criterion(...) then loss.backward(), as Executor.train
runs it), at the recipes' sizes: max_pooling B = 256, T = 300, D = 2; ce 4096 x 11; ctc B = 256, T <= 1000, V = 2599,
labels up to 200 tokens.  For each: the device criterion (wekws_b200.criterion) and torch's own ops on the same device
(the restatements of loss.py in oracle/kws_criterion*_oracle.py moved to CUDA, which is what runs without this
project).  Prints one JSON line with the card's name and power limit read in the same run, the p50 per step (host
clock around forward + backward ending in a device synchronise, after warm-up), the peak extra device memory of a
step (torch.cuda.max_memory_allocated over the step minus what was allocated before it), and for ctc_grad_kernel its
device time from torch.profiler and its share of the data sheet's 3.35 TB/s: the kernel is bound by HBM, and the
bytes it must move are the logits of the valid frames read once plus the whole gradient written once.
      python scripts/bench_criterion_grad.py [--iters 20]"""
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
from scripts.bench_criterion import batch as ctc_batch  # noqa: E402
from wekws_b200 import criterion  # noqa: E402

HBM_BYTES_PER_S = 3.35e12            # H100 SXM data sheet


def torch_criterion(type, logits, target, lengths, target_lengths=None, min_duration=0):
    """loss.py's ops on the logits' device, accuracy included as criterion() computes it: the B x D loop of
    max_pooling_loss, F.cross_entropy + acc_frame, log_softmax + F.ctc_loss (no accuracy in training)."""
    if type == "max_pooling":
        return max_pooling_on_device(logits, target, lengths, min_duration)
    if type == "ce":
        return K.cross_entropy(logits, target)[0]
    return K.ctc_loss(logits, target, lengths, target_lengths)[0]


def max_pooling_on_device(logits, target, lengths, min_duration):
    """kws_criterion_grad_oracle.max_pooling_loss_graph with its mask built on the logits' device (target read on the host, as loss.py does)."""
    B, T, D = logits.shape
    mask = torch.arange(T, device=logits.device)[None, :] >= lengths[:, None]
    target = target.cpu()
    loss = 0.0
    for i in range(B):
        for j in range(D):
            if int(target[i]) == j:
                m = mask[i].clone()
                m[:min_duration] = True
                pooled = logits[i, :, j].masked_fill(m, 0.0).clamp(1e-8, 1.0).max()
            else:
                pooled = (1 - logits[i, :, j]).masked_fill(mask[i], 1.0).clamp(1e-8, 1.0).min()
            loss = loss + -torch.log(pooled)
    max_p, idx = logits.masked_fill(mask[:, :, None], 0.0).max(1)[0].max(1)              # the accuracy, loss.py:74-86
    max_p, idx = max_p.tolist(), idx.tolist()
    sum((max_p[i] > 0.5 and idx[i] == int(target[i])) or (max_p[i] < 0.5 and int(target[i]) < 0) for i in range(B))
    return loss / B


def measure(step, iters, warmup=3):
    """(p50 seconds per step, peak extra bytes of a step)."""
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step()
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2], extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_criterion_grad.py needs a CUDA device")
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(3)
    cases = {}
    x = torch.rand(256, 300, 2, generator=g, device=dev) ** 3
    lens = torch.randint(100, 301, (256,), generator=g, device=dev)
    lens[0] = 300
    cases["max_pooling"] = (x, torch.randint(-1, 2, (256,), generator=g, device=dev), lens, None)
    cases["ce"] = (torch.randn(4096, 11, generator=g, device=dev) * 4,
                   torch.randint(0, 11, (4096,), generator=g, device=dev), None, None)
    B, T, V, L = 256, 1000, 2599, 200
    cx, ctgt, clens, ctl = ctc_batch(B, T, V, L, 7, dev)
    cases["ctc"] = (cx, ctgt, clens, ctl)

    out = {}
    for name, (x, tgt, lens, tl) in cases.items():
        x.requires_grad_(True)

        def ours():
            x.grad = None
            criterion(name, x, tgt, lens, tl)[0].backward()

        def theirs():
            x.grad = None
            torch_criterion(name, x, tgt, lens, tl).backward()

        t_ours, m_ours = measure(ours, args.iters)
        t_torch, m_torch = measure(theirs, args.iters if name != "max_pooling" else max(3, args.iters // 4))
        out[name] = {"p50_ms_device_criterion": round(t_ours * 1e3, 3), "p50_ms_torch_ops": round(t_torch * 1e3, 3),
                     "peak_extra_MB_device_criterion": round(m_ours / 1e6, 1),
                     "peak_extra_MB_torch_ops": round(m_torch / 1e6, 1)}

    x, tgt, lens, tl = cases["ctc"]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            x.grad = None
            criterion("ctc", x, tgt, lens, tl)[0].backward()
        torch.cuda.synchronize()
    kern = {}
    for k in ("ctc_row_kernel", "ctc_alpha_kernel", "ctc_beta_kernel", "ctc_grad_kernel"):
        ev = [e for e in prof.key_averages() if k in e.key]
        if not ev:
            raise SystemExit(f"bench_criterion_grad.py: {k} not found in the profile")
        kern[k] = sum(e.device_time_total for e in ev) / sum(e.count for e in ev) / 1e3          # ms per launch
    frames = int(lens.sum())
    grad_bytes = frames * V * 4 + B * T * V * 4          # valid logits rows read once + every gradient row written once
    rate = grad_bytes / (kern["ctc_grad_kernel"] * 1e-3)

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    gpu, power = (q[0].split(", ") + ["?"])[:2] if q else (torch.cuda.get_device_name(0), "?")
    print(json.dumps({
        "bench": "criterion_forward_backward", "gpu": gpu, "power_limit": power, "iters": args.iters,
        "sizes": {"max_pooling": [256, 300, 2], "ce": [4096, 11], "ctc": [B, T, V], "ctc_label_max": L,
                  "ctc_frames": frames},
        "steps": out, "ctc_kernel_ms": {k: round(v, 4) for k, v in kern.items()},
        "ctc_grad_kernel_bytes": grad_bytes, "ctc_grad_kernel_GBps": round(rate / 1e9, 1),
        "ctc_grad_kernel_share_of_3.35TBps": round(rate / HBM_BYTES_PER_S, 3),
    }))


if __name__ == "__main__":
    main()
