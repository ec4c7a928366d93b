#!/usr/bin/env python
"""Golden vectors for the global CMVN statistics (test infrastructure): drives the REFERENCE's own
tools/compute_cmvn_stats.py (its ``__main__``, through runpy) on a scripted wav.scp and writes
tests/golden/cmvn_stats.npz.

torchaudio 2.11 has no ``torchaudio.info`` and its ``load`` needs torchcodec, so exactly those two are replaced by
stubs that serve the scripted waveforms of oracle/kws_cmvn_oracle.py by path (int16 / 32768, as ``load`` normalises
PCM16).  The real ``Resample``, ``kaldi.fbank`` and ``kaldi.mfcc`` run; the two feature functions are wrapped only
to record the float64 sums of the features they return.  The DataLoader shuffle is seeded, num_workers is 0.

Per config <c> in fbank40, fbank80, mfcc80 (resample_rate 16000, every rate of oracle RATES, plain and segmented
lines): <c>_json the file the tool wrote, <c>_sum64 (2, D) the float64 sums of the reference's own features,
<c>_frames.  Per rate r != 16000: rs_in_<r> an int16 row, rs_ta_<r> torchaudio's Resample(r, 16000) of it and
rs_f64_<r> its float64 evaluation.  short_error: the exception the tool raises on an utterance shorter than one
400-sample frame after resampling.
      python oracle/make_cmvn_golden.py"""
import json
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFERENCE = "/root/reference"
TOOL = os.path.join(REFERENCE, "tools", "compute_cmvn_stats.py")
OUT = os.path.join(ROOT, "tests", "golden", "cmvn_stats.npz")
CONFIGS = {"fbank40": ("fbank", 40), "fbank80": ("fbank", 80), "mfcc80": ("mfcc", 80)}

from oracle import kws_cmvn_oracle as CO  # noqa: E402


class ScriptedAudio:
    """Replaces torchaudio.info / torchaudio.load with scripted waveforms keyed by path; records what was read."""

    def __init__(self, waves):
        self.waves = waves            # path -> (int16 array, rate)
        self.seen = set()

    def info(self, path, backend=None):
        return types.SimpleNamespace(sample_rate=self.waves[path][1])

    def load(self, filepath, frame_offset=0, num_frames=-1, normalize=True, channels_first=True, format=None,
             buffer_size=4096, backend=None):
        wav, rate = self.waves[filepath]
        seg = num_frames != -1
        end = len(wav) if not seg else frame_offset + num_frames
        self.seen.add((rate, "seg" if seg else "plain"))
        return torch.from_numpy(wav[frame_offset:end].astype(np.float32) / 32768.0)[None], rate


def run_tool(scp_lines, waves, feat_type, feat_dim, workdir):
    import torchaudio
    import torchaudio.compliance.kaldi as kaldi
    audio = ScriptedAudio(waves)
    sums = {"s": torch.zeros(2, feat_dim, dtype=torch.float64), "n": 0}
    real = {"fbank": kaldi.fbank, "mfcc": kaldi.mfcc, "info": getattr(torchaudio, "info", None),
            "load": torchaudio.load}

    def wrap(fn):
        def f(*a, **k):
            sums["depth"] = sums.get("depth", 0) + 1      # kaldi.mfcc calls kaldi.fbank: record the outer call only
            try:
                mat = fn(*a, **k)
            finally:
                sums["depth"] -= 1
            if sums["depth"]:
                return mat
            sums["s"][0] += mat.double().sum(0)
            sums["s"][1] += mat.double().square().sum(0)
            sums["n"] += mat.shape[0]
            return mat
        return f

    cfg = os.path.join(workdir, "train.yaml")
    with open(cfg, "w") as f:
        f.write(f"dataset_conf:\n    resample_conf:\n        resample_rate: 16000\n    feats_type: '{feat_type}'\n"
                f"    {feat_type}_conf:\n        num_mel_bins: {feat_dim}\n        dither: 1.0\n")
    scp = os.path.join(workdir, "wav.scp")
    with open(scp, "w") as f:
        f.write("".join(line + "\n" for line in scp_lines))
    out = os.path.join(workdir, "global_cmvn")
    argv = sys.argv
    try:
        kaldi.fbank, kaldi.mfcc = wrap(real["fbank"]), wrap(real["mfcc"])
        torchaudio.info, torchaudio.load = audio.info, audio.load
        sys.argv = [TOOL, "--train_config", cfg, "--in_scp", scp, "--out_cmvn", out, "--num_workers", "0"]
        torch.manual_seed(20240)
        runpy.run_path(TOOL, run_name="__main__")
    finally:
        sys.argv = argv
        kaldi.fbank, kaldi.mfcc, torchaudio.load = real["fbank"], real["mfcc"], real["load"]
        if real["info"] is None:
            del torchaudio.info
        else:
            torchaudio.info = real["info"]
    with open(out) as f:
        text = f.read()
    return text, sums["s"].numpy(), sums["n"], audio.seen


def main():
    import torchaudio
    utts = CO.golden_utterances()
    waves, lines = {}, []
    for i, (key, rate, n, seg) in enumerate(utts):
        path = f"/scripted/{key}.wav"
        waves[path] = (CO.utterance_wave(i, n), rate)
        lines.append(f"{key} {path}" if seg is None else f"{key} {path},{seg[0]},{seg[1]}")
    out = {"scp": np.array("\n".join(lines))}
    with tempfile.TemporaryDirectory() as d:
        for name, (ft, dim) in CONFIGS.items():
            text, s64, n, seen = run_tool(lines, waves, ft, dim, d)
            assert seen == {(r, k) for r in CO.RATES for k in ("plain", "seg")}, seen

            assert json.loads(text)["frame_num"] == n, (json.loads(text)["frame_num"], n)
            out[f"{name}_json"], out[f"{name}_sum64"], out[f"{name}_frames"] = np.array(text), s64, np.array(n)
            print(name, "frames", n)
        short = {"/scripted/short.wav": (CO.scripted_wave(7, 390), 16000)}
        try:
            run_tool(["short /scripted/short.wav"], short, "fbank", 40, d)
        except Exception as e:          # kaldi.fbank's assertion on a waveform shorter than one frame
            out["short_error"] = np.array(f"{type(e).__name__}: {e}")
        else:
            raise SystemExit("the tool accepted a 390-sample utterance")
    for i, rate in enumerate(r for r in CO.RATES if r != 16000):
        x = CO.scripted_wave(2000 + i, 2345 + 111 * i)
        xt = torch.from_numpy(x.astype(np.float32))
        ta = torchaudio.transforms.Resample(rate, 16000)(xt[None])[0]
        out[f"rs_in_{rate}"] = x
        out[f"rs_ta_{rate}"] = ta.numpy()
        out[f"rs_f64_{rate}"] = CO.resample(xt, rate, 16000, torch.float64).numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes;", out["short_error"])


if __name__ == "__main__":
    main()
