#!/usr/bin/env python
"""Times the training front-end (wekws_b200.TrainFeatures) at the recipes' batch sizes: 256 utterances of 1-2 s of
int16 audio at 16 kHz for the ds_tcn (fbank 40) and fsmn_ctc (fbank 80, context 2 / 2, frame skip 3) configs, 100 for
mdtc (mfcc 80).  Prints one JSON line with the card's name and power limit and, per config:
  * the Fbank / MFCC kernel's time per batch undithered and dithered (CUDA events around --reps launches);
  * the p50 of a whole TrainFeatures call (host clock around the call and a device synchronise);
  * the reference chain on one host core (kaldi.fbank / kaldi.mfcc with dither 1.0, processor.spec_aug's masking,
    context expansion and frame skip, restated with torch ops), timed on --cpu-utts utterances and extrapolated to the
    batch.
      python scripts/bench_train_features.py [--reps 50]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from wekws_b200 import TrainFeatures  # noqa: E402

CONFIGS = {
    "ds_tcn": (256, {"feats_type": "fbank", "fbank_conf": {"num_mel_bins": 40, "frame_shift": 10, "frame_length": 25,
                                                          "dither": 1.0},
                     "spec_aug": True, "spec_aug_conf": {"num_t_mask": 1, "num_f_mask": 1, "max_t": 20, "max_f": 10}}),
    "fsmn_ctc": (256, {"feats_type": "fbank", "fbank_conf": {"num_mel_bins": 80, "frame_shift": 10, "frame_length": 25,
                                                            "dither": 1.0},
                       "context_expansion": True, "context_expansion_conf": {"left": 2, "right": 2}, "frame_skip": 3,
                       "spec_aug": True, "spec_aug_conf": {"num_t_mask": 1, "num_f_mask": 1, "max_t": 20,
                                                           "max_f": 10}}),
    "mdtc": (100, {"feature_extraction_conf": {"feature_type": "mfcc", "num_ceps": 80, "num_mel_bins": 80,
                                               "frame_shift": 10, "frame_length": 25, "dither": 1.0},
                   "spec_aug": True, "spec_aug_conf": {"num_t_mask": 1, "num_f_mask": 1, "max_t": 20, "max_f": 40}}),
}


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def reference_chain(wav, conf, mfcc):
    """One utterance through the reference's worker chain (processor.py compute_* -> spec_aug -> context_expansion ->
    frame_skip), with the same torchaudio calls."""
    import torchaudio.compliance.kaldi as kaldi
    fc = conf.get("fbank_conf") or conf["feature_extraction_conf"]
    if mfcc:
        y = kaldi.mfcc(wav, num_ceps=80, num_mel_bins=80, frame_length=25, frame_shift=10, dither=1.0,
                       energy_floor=0.0, sample_frequency=16000)
    else:
        y = kaldi.fbank(wav, num_mel_bins=fc["num_mel_bins"], frame_length=25, frame_shift=10, dither=1.0,
                        energy_floor=0.0, sample_frequency=16000)
    y = y.clone().detach()
    sa = conf["spec_aug_conf"]
    for _ in range(sa["num_t_mask"]):
        s = random.randint(0, y.size(0) - 1)
        y[s:min(y.size(0), s + random.randint(1, sa["max_t"])), :] = 0
    for _ in range(sa["num_f_mask"]):
        s = random.randint(0, y.size(1) - 1)
        y[:, s:min(y.size(1), s + random.randint(1, sa["max_f"]))] = 0
    if conf.get("context_expansion"):
        left, right = conf["context_expansion_conf"]["left"], conf["context_expansion_conf"]["right"]
        ctx = torch.zeros(y.shape[0], y.shape[1] * (left + right + 1))
        for i, lag in enumerate(range(-left, right + 1)):
            ctx[:, i * y.shape[1]:(i + 1) * y.shape[1]] = torch.roll(y, -lag, 0)
        for idx in range(left):
            for cpx in range(left - idx):
                ctx[idx, cpx * y.shape[1]:(cpx + 1) * y.shape[1]] = ctx[left, :y.shape[1]]
        y = ctx[:ctx.shape[0] - right]
    return y[::conf.get("frame_skip", 1)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--cpu-utts", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_features.py needs a CUDA device")
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    result = {"card": torch.cuda.get_device_name(dev), "nvidia_smi": smi[0] if smi else None, "configs": {}}
    torch.set_num_threads(1)
    for name, (B, conf) in CONFIGS.items():
        g = torch.Generator().manual_seed(0)
        lens = torch.randint(16000, 32001, (B,), generator=g).tolist()
        pcm = (torch.randn(B, max(lens), generator=g) * 2000).round().to(torch.int16)
        x = pcm.to(dev)
        tf = TrainFeatures.from_config(conf)
        fe, d_lens = tf.frontend, torch.tensor(lens, dtype=torch.int32, device=dev)
        out = torch.empty(B, fe.num_frames(max(lens)), fe.feature_dim, device=dev)
        plain = event_ms(lambda: fe(x, lengths=d_lens, out=out), args.reps)
        dith = event_ms(lambda: fe(x, lengths=d_lens, out=out, dither=1.0), args.reps)
        labels, keys = [0] * B, [str(i) for i in range(B)]
        call = lambda: tf(x, lens, 16000, labels, keys)      # noqa: E731
        call()
        times = []
        for _ in range(max(10, args.reps // 2)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            call()
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        p50 = sorted(times)[len(times) // 2]
        n = min(args.cpu_utts, B)
        reference_chain(pcm[:1, :lens[0]].float(), conf, name == "mdtc")      # torchaudio's first-call set-up
        t0 = time.perf_counter()
        for b in range(n):
            reference_chain(pcm[b:b + 1, :lens[b]].float(), conf, name == "mdtc")
        cpu_per_utt = (time.perf_counter() - t0) / n
        audio_s = sum(lens) / 16000.0
        result["configs"][name] = {
            "batch": B, "audio_s": round(audio_s, 1),
            "kernel_ms_undithered": round(plain, 4), "kernel_ms_dithered": round(dith, 4),
            "dither_cost": round(dith / plain, 2),
            "train_features_p50_ms": round(p50 * 1e3, 3),
            "reference_one_core_ms_per_batch": round(cpu_per_utt * B * 1e3, 1),
            "reference_one_core_ms_per_audio_s": round(cpu_per_utt * B * 1e3 / audio_s, 3),
        }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
