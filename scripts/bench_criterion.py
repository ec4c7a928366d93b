#!/usr/bin/env python
"""Times the CTC validation criterion (wekws_b200.criterion('ctc', ..., validation=True), as Executor.cv calls it) at
the recipe's size: B = 256 utterances, T <= 1000 frames, V = 2599 tokens, labels up to 200 tokens.  Prints one JSON
line with the card's name and power limit, the p50 per batch (host clock around the call, which ends in a device
synchronise, after warm-up) with and without validation, the HBM rate of the logits pass (ctc_row_kernel's device
time from torch.profiler over the bytes it must read), and the CPU restatement of the reference on a few
utterances, extrapolated to the batch.
      python scripts/bench_criterion.py [--iters 20]"""
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
from wekws_b200 import criterion  # noqa: E402


def batch(B, T, V, L, seed, dev):
    """Peaky logits that spell the first 30 tokens of each label (blank on every third frame) over N(0, 1)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    lens = torch.randint(T // 2, T + 1, (B,), generator=g, device=dev)
    lens[0] = T
    tl = torch.randint(1, L + 1, (B,), generator=g, device=dev)
    tgt = torch.randint(1, V, (B, L), generator=g, device=dev)
    tgt[torch.arange(L, device=dev)[None, :] >= tl[:, None]] = -1
    x = torch.randn(B, T, V, generator=g, device=dev)
    t = torch.arange(T, device=dev)[None, :]
    spelled = tl.clamp(max=30)[:, None]
    pos = (t * spelled // lens[:, None]).clamp(max=spelled - 1)
    hot = torch.where(t % 3 == 2, torch.zeros_like(pos), tgt.gather(1, pos))
    x.scatter_add_(2, hot[:, :, None], torch.full((B, T, 1), 9.0, device=dev))
    return x, tgt, lens, tl


def p50(fn, iters):
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--cpu-utts", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_criterion.py needs a CUDA device")
    dev = torch.device("cuda:0")
    B, T, V, L = 256, 1000, 2599, 200
    x, tgt, lens, tl = batch(B, T, V, L, 7, dev)

    def val():
        return criterion("ctc", x, tgt, lens, tl, validation=True)

    def loss_only():
        return criterion("ctc", x, tgt, lens, tl, validation=False)

    for _ in range(3):
        val()
        loss_only()
    torch.cuda.synchronize()
    t_val = p50(val, args.iters)
    t_loss = p50(loss_only, args.iters)

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            val()
        torch.cuda.synchronize()
    kern = {}
    for name in ("ctc_row_kernel", "ctc_alpha_kernel", "ctc_prefix_beam_kernel", "ctc_edit_kernel",
                 "criterion_reduce_kernel"):
        ev = [e for e in prof.key_averages() if name in e.key]
        if not ev:
            raise SystemExit(f"bench_criterion.py: {name} not found in the profile")
        kern[name] = sum(e.device_time_total for e in ev) / sum(e.count for e in ev) / 1e3      # ms per launch
    row_ms = kern["ctc_row_kernel"]
    frames = int(lens.sum())
    row_bytes = frames * V * 4                           # the valid rows of the logits, read once by the row pass

    n = args.cpu_utts
    xc, tc, lc, tlc = x[:n].cpu(), tgt[:n].cpu(), lens[:n].cpu(), tl[:n].cpu()
    t0 = time.perf_counter()
    K.criterion("ctc", xc, tc, lc, tlc, validation=True)
    cpu_s = (time.perf_counter() - t0) * B / n

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else (torch.cuda.get_device_name(0), "?")
    print(json.dumps({
        "bench": "criterion_ctc_validation", "gpu": name, "power_limit": power, "B": B, "T_max": T, "V": V,
        "label_max": L, "frames": frames, "p50_ms_validation": round(t_val * 1e3, 3),
        "p50_ms_loss_only": round(t_loss * 1e3, 3),
        "kernel_ms": {k: round(v, 4) for k, v in kern.items()},
        "row_pass_GBps": round(row_bytes / (row_ms * 1e-3) / 1e9, 1),
        "cpu_reference_restatement_s_extrapolated": round(cpu_s, 2), "cpu_utts_timed": n,
    }))


if __name__ == "__main__":
    main()
