#!/usr/bin/env python
"""Times the training-audio augmentation (wekws_b200.reverb / add_noise) on a recipe-sized batch: 256 rows of 1-3 s
of int16 audio at 16 kHz, every row selected (probability 1.0), with a bank of 8000-tap and one of 16000-tap RIRs.
Prints one JSON line with the card's name, power limit and maximum SM clock and, per RIR length:
  * ms per batch of the reverb and of the noise call (host clock around --reps calls and a device synchronise: the
    draws, the upload and the launch), and of the reverb kernel alone (CUDA events around --reps launches);
  * the reverb's useful multiply-adds (sum over rows of sum_i min(i + 1, taps)) per second, against the card's FP64
    FMA peak (SMs x 64 FP64 FMAs per clock x the maximum SM clock);
  * the reference's arithmetic on one host core (processor.add_reverb's scipy.signal.convolve of float32 rows,
    processor.add_noise's numpy), timed on --cpu-rows rows after one warm-up call and extrapolated to the batch.
      python scripts/bench_augment.py [--reps 10]"""
import argparse
import ctypes as C
import io
import json
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from wekws_b200 import AugmentSource, _native, add_noise, reverb  # noqa: E402
from wekws_b200.augment import _upload, draw_reverb  # noqa: E402


def wav(a):
    from scipy.io import wavfile
    f = io.BytesIO()
    wavfile.write(f, 16000, a)
    return f.getvalue()


def host_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def reference_reverb(x, rir):
    from scipy import signal
    rir = rir / np.sqrt(np.sum(rir ** 2))
    return signal.convolve(x, rir, mode="full")[:x.shape[0]]


def reference_noise(x, s, snr):
    audio_db = 10 * np.log10(np.mean(x ** 2) + 1e-4)
    noise_db = 10 * np.log10(np.mean(s ** 2) + 1e-4)
    return x + np.sqrt(10 ** ((audio_db - noise_db - snr) / 10)) * s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cpu-rows", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment.py needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    props = torch.cuda.get_device_properties(dev)
    max_mhz = None
    if smi:
        try:
            max_mhz = float(smi[0].split(",")[2].strip().split()[0])
        except (IndexError, ValueError):
            pass
    peak = props.multi_processor_count * 64 * max_mhz * 1e6 if max_mhz else None
    result = {"card": torch.cuda.get_device_name(dev), "nvidia_smi": smi[0] if smi else None,
              "fp64_fma_peak_per_s": peak, "rir": {}}
    torch.set_num_threads(1)
    B = 256
    g = np.random.default_rng(0)
    lens = [int(v) for v in g.integers(16000, 48001, B)]
    pcm = np.zeros((B, max(lens)), np.int16)
    for b, n in enumerate(lens):
        pcm[b, :n] = np.clip(np.round(g.standard_normal(n) * 2000), -32768, 32767)
    x = torch.from_numpy(pcm).to(dev)
    noise = AugmentSource([(f"{p}_{i}", wav(np.round(g.standard_normal(int(g.integers(8000, 160000))) * 3000)
                                            .astype(np.int16)))
                           for i, p in enumerate(["noise", "speech", "music"] * 4)])
    nz_ms = host_ms(lambda: add_noise(x, lens, noise, 1.0, rng=random.Random(1)), args.reps)
    n = min(args.cpu_rows, B)
    reference_reverb(pcm[0, :lens[0]].astype(np.float32), np.ones(8000, np.float32))     # scipy's first-call set-up
    t0 = time.perf_counter()
    for b in range(n):
        xb = pcm[b, :lens[b]].astype(np.float32) / 32768
        s = noise.clips[b % len(noise)]
        s = s[:lens[b]] if s.size > lens[b] else np.resize(s, (lens[b],))
        reference_noise(xb, s, 10.0)
    cpu_nz = (time.perf_counter() - t0) / n * B * 1e3
    result["noise"] = {"batch": B, "audio_s": round(sum(lens) / 16000, 1), "ms_per_batch": round(nz_ms, 3),
                       "reference_one_core_ms_per_batch": round(cpu_nz, 1)}
    for taps in (8000, 16000):
        rirs = AugmentSource([(f"rir_{i}", wav((g.standard_normal(taps) * np.exp(-np.arange(taps) / (taps / 5)))
                                               .astype(np.float32))) for i in range(8)], rir=True)
        call_ms = host_ms(lambda: reverb(x, lens, rirs, 1.0, rng=random.Random(2)), args.reps)
        r = random.Random(2)
        picks = [draw_reverb(n_, rirs, 1.0, r, b) for b, n_ in enumerate(lens)]
        # the kernel alone: the same launch with the table already on the device
        offsets, clips, rows, nf = {}, [], [], 0
        for b, i in enumerate(picks):
            if i not in offsets:
                offsets[i] = nf
                clips.append(rirs.clips[i])
                nf += rirs.lengths[i]
            rows += [lens[b], offsets[i], rirs.lengths[i]]
        d, o_rows, o_clip = _upload(dev, rows, clips)
        out = torch.empty(B, x.shape[1], device=dev)
        st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)

        def launch():
            _native.check(_native.lib().wekws_reverb(C.c_void_p(x.data_ptr()), _native.PCM_S16, B, x.shape[1],
                                                     x.stride(0), C.c_void_p(d.data_ptr() + o_rows),
                                                     C.c_void_p(d.data_ptr() + o_clip), C.c_void_p(out.data_ptr()),
                                                     out.stride(0), st), "wekws_reverb")
        launch()
        torch.cuda.synchronize()
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            launch()
        e.record()
        torch.cuda.synchronize()
        kern_ms = a.elapsed_time(e) / args.reps
        macs = sum(min(n_, taps) * (min(n_, taps) + 1) // 2 + max(0, n_ - taps) * taps for n_ in lens)
        t0 = time.perf_counter()
        for b in range(n):
            reference_reverb(pcm[b, :lens[b]].astype(np.float32) / 32768, rirs.clips[picks[b]])
        cpu_rv = (time.perf_counter() - t0) / n * B * 1e3
        rate = macs / (kern_ms * 1e-3)
        result["rir"][str(taps)] = {
            "batch": B, "reverb_call_ms_per_batch": round(call_ms, 3), "reverb_kernel_ms": round(kern_ms, 3),
            "useful_gmac": round(macs / 1e9, 2), "gmac_per_s": round(rate / 1e9, 1),
            "share_of_fp64_fma_peak": round(rate / peak, 3) if peak else None,
            "reference_one_core_ms_per_batch": round(cpu_rv, 1)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
