"""CPU oracle for the global CMVN statistics of tools/compute_cmvn_stats.py (TEST INFRASTRUCTURE ONLY; nothing in
``wekws_b200/`` imports it).

* ``resample_kernel`` / ``resample`` restate torchaudio 2.11's ``_get_sinc_resample_kernel`` (sinc_interp_hann) and
  ``_apply_sinc_resample_kernel`` with the same torch ops, so on the CPU they are bit-identical to
  ``torchaudio.transforms.Resample`` (pinned by tests/test_cmvn_stats_host.py whenever torchaudio imports).  With
  dtype=float64 the float32 table and the waveform are evaluated in double: the yardstick the device resampler is
  ranked against.
* ``collate`` restates ``CollateFunc.__call__`` (compute_cmvn_stats.py:26-72) on in-memory waveforms, with this
  module's resampler and kws_oracle's ``fbank`` / ``mfcc``: the float32 accumulators of the tool, and alongside them
  the float64 sums of the same float32 features.  ``collate(..., dtype=torch.float64)`` runs the whole chain in
  double (the truth the statistics tests measure errors against).
* ``scripted_wave`` is the deterministic int16 audio the golden generator and the tests share.
"""
from __future__ import annotations

import math
from typing import List, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import kws_oracle as O

Tensor = torch.Tensor


def resample_kernel(orig_freq: int, new_freq: int, lowpass_filter_width: int = 6, rolloff: float = 0.99):
    """torchaudio functional.py `_get_sinc_resample_kernel` (dtype None, Hann window): (new/g, 1, K) float32, width."""
    gcd = math.gcd(int(orig_freq), int(new_freq))
    orig_freq, new_freq = int(orig_freq) // gcd, int(new_freq) // gcd
    base_freq = min(orig_freq, new_freq) * rolloff
    width = math.ceil(lowpass_filter_width * orig_freq / base_freq)
    idx = torch.arange(-width, width + orig_freq, dtype=torch.float64)[None, None] / orig_freq
    t = torch.arange(0, -new_freq, -1, dtype=None)[:, None, None] / new_freq + idx
    t *= base_freq
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t *= math.pi
    scale = base_freq / orig_freq
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * scale
    return kernels.to(dtype=torch.float32), width


def resample(waveform: Tensor, orig_freq: int, new_freq: int, dtype=torch.float32) -> Tensor:
    """torchaudio `_apply_sinc_resample_kernel` on (..., N) (the input unchanged at equal rates, as the transform)."""
    if int(orig_freq) == int(new_freq):
        return waveform
    kernel, width = resample_kernel(orig_freq, new_freq)
    gcd = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // gcd, int(new_freq) // gcd
    shape = waveform.size()
    wav = waveform.to(dtype).reshape(-1, shape[-1])
    num_wavs, length = wav.shape
    wav = F.pad(wav, (width, width + orig))
    out = F.conv1d(wav[:, None], kernel.to(dtype), stride=orig)
    out = out.transpose(1, 2).reshape(num_wavs, -1)
    target = torch.ceil(torch.as_tensor(new * length / orig)).long()
    out = out[..., :target]
    return out.view(shape[:-1] + out.shape[-1:])


def resample_abs_bound(waveform: Tensor, orig_freq: int, new_freq: int) -> Tensor:
    """sum_k |kernel| |x| per output (float64): 2^-52 of it bounds how far two double evaluations of one output can
    differ with different summation orders (a few dozen terms)."""
    kernel, width = resample_kernel(orig_freq, new_freq)
    gcd = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // gcd, int(new_freq) // gcd
    wav = waveform.to(torch.float64).reshape(1, -1).abs()
    length = wav.shape[-1]
    wav = F.pad(wav, (width, width + orig))
    out = F.conv1d(wav[:, None], kernel.to(torch.float64).abs(), stride=orig).transpose(1, 2).reshape(-1)
    return out[:math.ceil(new * length / orig)]


def scripted_wave(seed: int, n: int) -> np.ndarray:
    """Deterministic int16 test audio: two tones and amplitude-modulated noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n, dtype=np.float64)
    f1, f2 = rng.uniform(0.002, 0.03), rng.uniform(0.05, 0.2)
    x = (2500 * np.sin(2 * np.pi * f1 * t) + 800 * np.sin(2 * np.pi * f2 * t + 1.0)
         + 1500 * rng.standard_normal(n) * (0.3 + 0.7 * np.abs(np.sin(np.pi * t / max(n, 1) * 3))))
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def features(wav: Tensor, feat_type: str, feat_dim: int, sample_rate: int, dtype=torch.float32) -> Tensor:
    """kaldi.fbank / kaldi.mfcc with the tool's arguments (compute_cmvn_stats.py:54-68)."""
    if feat_type == "fbank":
        return O.fbank(wav, num_mel_bins=feat_dim, sample_frequency=sample_rate, dtype=dtype)
    if feat_type == "mfcc":
        return O.mfcc(wav, num_ceps=feat_dim, num_mel_bins=feat_dim, sample_frequency=sample_rate, dtype=dtype)
    raise ValueError(feat_type)


def collate(items: Sequence[Tuple[Tensor, int]], feat_type: str, feat_dim: int, resample_rate: int,
            dtype=torch.float32):
    """CollateFunc.__call__ on [(waveform (N,) at int16 scale, sample_rate)].  Returns (number, mean_stat, var_stat,
    sum64) where mean_stat / var_stat are accumulated as the tool does (in `dtype`) and sum64 (2, D) float64 are the
    sums of the same features in double."""
    mean_stat = torch.zeros(feat_dim, dtype=dtype)
    var_stat = torch.zeros(feat_dim, dtype=dtype)
    sum64 = torch.zeros(2, feat_dim, dtype=torch.float64)
    number = 0
    for wav, sr in items:
        wav = wav.to(dtype)
        rate = sr
        if resample_rate != 0 and resample_rate != sr:
            rate = resample_rate
            wav = resample(wav, sr, rate, dtype)
        if wav.numel() < 400:
            raise AssertionError("choose a window size 400 that is [2, %d]" % wav.numel())
        mat = features(wav, feat_type, feat_dim, rate, dtype)
        mean_stat += torch.sum(mat, axis=0)
        var_stat += torch.sum(torch.square(mat), axis=0)
        sum64[0] += mat.double().sum(0)
        sum64[1] += mat.double().square().sum(0)
        number += mat.shape[0]
    return number, mean_stat, var_stat, sum64


# the utterances of tests/golden/cmvn_stats.npz: (key, rate, samples in the file, segment (start s, end s) or None)
RATES = (8000, 11025, 16000, 22050, 44100, 48000)


def golden_utterances() -> List[Tuple[str, int, int, object]]:
    out = []
    for i, rate in enumerate(RATES):
        out.append((f"plain{rate}", rate, int(rate * (0.55 + 0.07 * i)), None))
        out.append((f"seg{rate}", rate, int(rate * 1.1), (0.13 + 0.01 * i, 0.81 + 0.02 * i)))
        out.append((f"brief{rate}", rate, int(rate * 0.3) + 7 * i, None))
    return out


def utterance_wave(index: int, n: int) -> np.ndarray:
    return scripted_wave(1000 + index, n)
