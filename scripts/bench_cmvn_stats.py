#!/usr/bin/env python
"""Times the global CMVN statistics (wekws_b200.CmvnStats.update, the device twin of tools/compute_cmvn_stats.py) on
synthetic training sets: --utts utterances of 1-5 s of int16 audio at 16 kHz and at 48 kHz (resampled to 16 kHz),
fbank 80, batches of --batch.  Prints one JSON line with the card's name and power limit and, per rate:
  * utterance-hours per second of the whole update (resample + Fbank + statistics), and of the resampler alone;
  * each kernel's share of the device time (torch.profiler), so the cost of the separate statistics pass is visible;
  * the resampler's achieved input rate (valid int16 samples it reads / its device time);
  * the reference's CollateFunc restated on one host core (oracle/kws_cmvn_oracle.py collate, float32 as the tool)
    timed on --cpu-utts utterances and extrapolated to the set.
      python scripts/bench_cmvn_stats.py [--utts 2000] [--batch 250]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import kws_cmvn_oracle as CO  # noqa: E402
from wekws_b200 import CmvnStats, Resample  # noqa: E402

KERNELS = ("resample_kernel", "fbank_kernel", "cmvn_utt_sums_kernel", "cmvn_fold_kernel")


def make_set(rate, utts, batch, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for i in range(0, utts, batch):
        b = min(batch, utts - i)
        lens = torch.randint(rate, 5 * rate + 1, (b,), generator=g, device=dev)
        pcm = (torch.randn(b, int(lens.max()), generator=g, device=dev) * 2000).round().to(torch.int16)
        out.append((pcm, lens.tolist()))
    return out


def timed(fn, reps):
    best = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best.append(time.perf_counter() - t0)
    return sorted(best)[len(best) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=250)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-utts", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cmvn_stats.py needs a CUDA device")
    dev = torch.device("cuda:0")
    res = {}
    for rate in (16000, 48000):
        data = make_set(rate, args.utts, args.batch, 3 + rate, dev)
        seconds = sum(sum(lens) for _, lens in data) / rate

        st = CmvnStats("fbank", 80, resample_rate=16000)       # handles and tables are built on the first update

        def full():
            for pcm, lens in data:
                st.update(pcm, lens, rate)

        full()
        t_full = timed(full, args.reps)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            full()
            torch.cuda.synchronize()
        kern = {k: sum(e.device_time_total for e in prof.key_averages() if k in e.key) / 1e3 for k in KERNELS}
        r = {"audio_hours": round(seconds / 3600, 3), "update_s": round(t_full, 4),
             "update_utt_hours_per_s": round(seconds / 3600 / t_full, 1),
             "kernel_ms": {k: round(v, 3) for k, v in kern.items() if v > 0}}
        if rate != 16000:
            rs = Resample(rate, 16000)
            lens_d = [torch.tensor(lens, device=dev) for _, lens in data]

            def resample_only():
                for (pcm, _), ld in zip(data, lens_d):
                    rs(pcm, ld)

            resample_only()
            t_rs = timed(resample_only, args.reps)
            r["resample_utt_hours_per_s"] = round(seconds / 3600 / t_rs, 1)
            r["resample_input_GBps"] = round(seconds * rate * 2 / (kern["resample_kernel"] * 1e-3) / 1e9, 1)
        torch.set_num_threads(1)
        pcm, lens = data[0]
        items = [(pcm[b, :lens[b]].float().cpu(), rate) for b in range(args.cpu_utts)]
        t0 = time.perf_counter()
        CO.collate(items, "fbank", 80, 16000)
        cpu = (time.perf_counter() - t0) / sum(len(w) for w, _ in items) * rate
        r["cpu_reference_one_core_s_per_audio_s"] = round(cpu, 5)
        r["cpu_reference_one_core_s_extrapolated"] = round(cpu * seconds, 1)
        res[f"{rate // 1000}k"] = r
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    name, power = (q[0].split(", ") + ["?"])[:2] if q else (torch.cuda.get_device_name(0), "?")
    print(json.dumps({"bench": "cmvn_stats", "gpu": name, "power_limit": power, "utts": args.utts,
                      "batch": args.batch, "feats": "fbank80", **res}))


if __name__ == "__main__":
    main()
