#!/usr/bin/env python
"""The training step's optimiser on the device against torch's, on the parameter sets of every shipped training model.

Per parameter set, p50 over --steps of clip_grad_norm_(max_norm 5) + Adam.step() (lr 1e-3) for torch.optim.Adam
(foreach, the default), torch.optim.Adam(fused=True), each after torch.nn.utils.clip_grad_norm_, and
wekws_b200.clip_grad_norm_ + wekws_b200.Adam:
  * host_ms: time until the calls return (what the Python thread spends);
  * device_ms: CUDA events around the calls, with the stream held busy by a queued sleep kernel so that the events
    measure the device work and not the host's enqueue gaps;
  * wall_ms: host clock around the calls ending in a synchronise.
Then the whole Executor.train step (forward, criterion("max_pooling"), backward, clip, step) of mdtc at B = 100,
T = 200 (scripts/bench_mdtc_train.py's shape) with each optimiser, and a torch.profiler breakdown of that step with
torch's default Adam and with ours (chrome traces under --trace-dir, a temporary directory by default).  Reports the
card and its power limit.  One JSON line.
      python scripts/bench_optim.py [--steps 50] [--warmup 10] [--trace-dir DIR]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.test_optim_host import PARAM_SETS  # noqa: E402
import wekws_b200  # noqa: E402
from wekws_b200 import criterion, init_model, model_config, synth  # noqa: E402

DEV = torch.device("cuda:0")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def p50(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


OPTIMISERS = {
    "torch_foreach": (lambda ps: torch.optim.Adam(ps, lr=1e-3), torch.nn.utils.clip_grad_norm_),
    "torch_fused": (lambda ps: torch.optim.Adam(ps, lr=1e-3, fused=True), torch.nn.utils.clip_grad_norm_),
    "ours": (lambda ps: wekws_b200.Adam(ps, lr=1e-3), wekws_b200.clip_grad_norm_),
}


def time_step(params, make_opt, clip, steps, warmup):
    opt = make_opt(params)
    gen = torch.Generator(device=DEV).manual_seed(1)
    grads = [torch.randn(p.shape, generator=gen, device=DEV) * 1e-2 for p in params]

    def run():
        clip(params, 5.0)
        opt.step()

    host, dev, wall = [], [], []
    for i in range(warmup + steps):
        for p, g in zip(params, grads):
            p.grad = g.clone()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        host.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        wall.append(time.perf_counter() - t0)
        # device time: the stream is parked on a sleep while the host enqueues, so the events bracket device work only
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(20_000_000)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        dev.append(e0.elapsed_time(e1) * 1e-3)
    ms = lambda xs: round(p50(xs[warmup:]) * 1e3, 4)
    return {"host_ms": ms(host), "device_ms": ms(dev), "wall_ms": ms(wall)}


def mdtc_step(make_opt, clip, steps, warmup, profile_dir=None):
    B, T = 100, 200
    model = synth.randomize_(init_model(model_config("mdtc")), seed=1).to(DEV).enable_training().train()
    gen = torch.Generator().manual_seed(2)
    feats = torch.randn(B, T, 80, generator=gen).to(DEV)
    lens = torch.randint(T // 2, T + 1, (B,), generator=gen).to(DEV)
    target = torch.randint(-1, 1, (B,), generator=gen).to(DEV)
    opt = make_opt(list(model.parameters()))

    def run():
        out, _ = model(feats)
        loss, acc = criterion("max_pooling", out, target, lens)
        opt.zero_grad()
        loss.backward()
        grad_norm = clip(model.parameters(), 5.0)
        if torch.isfinite(grad_norm):
            opt.step()

    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        t0 = time.perf_counter()
        run()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    res = round(p50(ts) * 1e3, 3)
    if profile_dir is None:
        return res, None
    from torch.profiler import ProfilerActivity, profile, record_function
    phases = {}

    def run_marked():
        with record_function("step.forward"):
            out, _ = model(feats)
        with record_function("step.criterion"):
            loss, acc = criterion("max_pooling", out, target, lens)
        with record_function("step.zero_grad"):
            opt.zero_grad()
        with record_function("step.backward"):
            loss.backward()
        with record_function("step.clip_grad_norm_"):
            grad_norm = clip(model.parameters(), 5.0)
        with record_function("step.isfinite"):
            ok = bool(torch.isfinite(grad_norm))
        if ok:
            with record_function("step.optimizer_step"):
                opt.step()

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            run_marked()
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if e.key.startswith("step."):
            phases[e.key] = {"cpu_ms_per_step": round(e.cpu_time_total / 10 / 1e3, 3),
                             "device_ms_per_step": round(getattr(e, "device_time_total", 0.0) / 10 / 1e3, 3)}
    os.makedirs(profile_dir, exist_ok=True)
    prof.export_chrome_trace(os.path.join(profile_dir, "mdtc_train_step_torch_adam.json"))
    return res, phases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--trace-dir", default=os.path.join(tempfile.gettempdir(), "wekws_bench_optim"))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_optim needs a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    out = {"card": card(), "torch": torch.__version__, "optimiser_step": {}, "executor_train_mdtc_100x200_ms": {}}
    for name, cfg in PARAM_SETS.items():
        base = [p.detach().to(DEV) for p in synth.randomize_(init_model(cfg()), seed=0).parameters()]
        row = {"tensors": len(base), "elements": sum(p.numel() for p in base)}
        for oname, (make_opt, clip) in OPTIMISERS.items():
            params = [torch.nn.Parameter(t.clone()) for t in base]
            row[oname] = time_step(params, make_opt, clip, a.steps, a.warmup)
        out["optimiser_step"][name] = row
    for oname, (make_opt, clip) in OPTIMISERS.items():
        t, _ = mdtc_step(make_opt, clip, a.steps, a.warmup)
        out["executor_train_mdtc_100x200_ms"][oname] = t
    _, phases = mdtc_step(*OPTIMISERS["torch_foreach"], 3, 3, profile_dir=a.trace_dir)
    out["profile_mdtc_step_torch_foreach"] = phases
    _, phases = mdtc_step(*OPTIMISERS["ours"], 3, 3, profile_dir=os.path.join(a.trace_dir, "ours"))
    out["profile_mdtc_step_ours"] = phases
    print(json.dumps(out))


if __name__ == "__main__":
    main()
