#!/usr/bin/env python
"""Global CMVN statistics of a training set on the GPU: a drop-in for the recipes' stage 1
(``tools/compute_cmvn_stats.py --num_workers 16 --train_config ... --in_scp ... --out_cmvn ...``).

Reads the wav.scp (``key path`` or ``key path,start_s,end_s`` lines), decodes PCM16 or float32 WAV files on the host
with scipy.io.wavfile, groups the utterances by sample rate into batches of --batch, feeds wekws_b200.CmvnStats
(resampling, Fbank / MFCC and the statistics on the device) and writes the global_cmvn JSON that init_model's
cmvn_file reads.  The sums are accumulated and written in double.  --num_workers is accepted for command-line
compatibility and ignored.
      python scripts/compute_cmvn_stats.py --train_config conf/ds_tcn.yaml --in_scp data/train/wav.scp \
          --out_cmvn data/train/global_cmvn"""
import argparse
import os
import sys

import numpy as np
import torch
import yaml
from scipy.io import wavfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from wekws_b200 import CmvnStats, scp_segment  # noqa: E402


def read_wav(path):
    """(rate, int16 or float32 samples at int16 scale) of channel 0 (kaldi.fbank's default channel)."""
    rate, data = wavfile.read(path)
    if data.ndim == 2:
        data = data[:, 0]
    if data.dtype == np.int16:
        return rate, data
    if data.dtype == np.float32:
        return rate, data * np.float32(1 << 15)
    raise SystemExit(f"compute_cmvn_stats.py: {path}: {data.dtype} WAV samples are not supported "
                     "(PCM16 or float32 WAV only)")


def scp_items(path):
    with open(path, encoding="utf-8") as f:
        for line in f:
            arr = line.strip().split()
            if arr:
                yield arr[0], arr[1]


def main():
    ap = argparse.ArgumentParser(description="extract CMVN stats on the GPU")
    ap.add_argument("--num_workers", default=0, type=int, help="ignored (decoding is cheap next to the tool's)")
    ap.add_argument("--train_config", default="", help="training yaml conf")
    ap.add_argument("--in_scp", default=None, help="wav scp file")
    ap.add_argument("--out_cmvn", default="global_cmvn", help="global cmvn file")
    ap.add_argument("--batch", default=64, type=int, help="utterances per device batch")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("compute_cmvn_stats.py needs a CUDA device")
    with open(args.train_config) as fin:
        configs = yaml.load(fin, Loader=yaml.FullLoader)
    stats = CmvnStats.from_config(configs)
    if stats.resample_rate:
        print(f"using resample and new sample rate is {stats.resample_rate}")
    dev = torch.device("cuda:0")
    pending = {}            # sample rate -> [samples]
    done = 0

    def flush(rate):
        nonlocal done
        wavs = pending.pop(rate)
        n = max(len(w) for w in wavs)
        dtype = torch.int16 if all(w.dtype == np.int16 for w in wavs) else torch.float32
        batch = torch.zeros(len(wavs), n, dtype=dtype)
        for i, w in enumerate(wavs):
            batch[i, :len(w)] = torch.from_numpy(np.ascontiguousarray(w)).to(dtype)
        stats.update(batch.to(dev), [len(w) for w in wavs], rate)
        done += len(wavs)
        print(f"processed {done} wavs, {stats.frame_num} frames", file=sys.stderr, flush=True)

    for key, value in scp_items(args.in_scp):
        path = value.strip().split(",")[0]
        rate, data = read_wav(path)
        _, start, end = scp_segment(value, rate)
        if start is not None:
            data = data[start:end]
        pending.setdefault(rate, []).append(data)
        if len(pending[rate]) >= args.batch:
            flush(rate)
    for rate in list(pending):
        flush(rate)
    stats.write(args.out_cmvn)


if __name__ == "__main__":
    main()
