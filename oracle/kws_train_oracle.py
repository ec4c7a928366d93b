"""CPU oracle of the training front-end (wekws_b200/train_features.py).  TEST INFRASTRUCTURE ONLY.

* ``philox4x32_10`` / ``dither_noise``: the dither generator of wekws_b200/csrc/dither.cuh restated in numpy, the
  Philox words bit for bit and the Box-Muller normals in float64.
* ``fbank`` / ``mfcc``: oracle/kws_oracle.py's restatements of kaldi.fbank / kaldi.mfcc with ``noise``, an (m, 400)
  tensor added to the framed signal where torchaudio adds torch.randn(m, 400) * dither (kaldi.py _get_window), before
  DC removal, pre-emphasis and the window.  With noise=None they are kws_oracle's functions.
* ``train_chain``: the reference's per-utterance training chain (compute_fbank / compute_mfcc with the restated noise,
  spec_aug, context_expansion, frame_skip), evaluated in float64 by default: the yardstick for features where the
  reference's own float32 rounding is above the feature tolerance.
* ``golden_audio`` / ``spec_aug_input``: the seeded inputs of tests/golden/train_features.npz, which stores only the
  reference's outputs (oracle/make_train_features_golden.py).
"""
from __future__ import annotations

import math
import random
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from oracle import kws_oracle as O

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr: np.ndarray, key) -> np.ndarray:
    """Philox4x32-10 of counters ctr (..., 4) uint32 with key (k0, k1): Random123's philox4x32 with 10 rounds."""
    c = [np.asarray(ctr[..., i], dtype=np.uint64) for i in range(4)]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & MASK32,
             (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & MASK32]
    return np.stack(c, axis=-1).astype(np.uint32)


def dither_noise(seed: int, B: int, frames: int, win: int = 400) -> np.ndarray:
    """(B, frames, win) float64 normals: counter (j // 4, f, b, 0), key (seed lo, seed hi); words (x0..x3) give
    samples 4q..4q+3 as (r cos 2 pi u1, r sin 2 pi u1, r' cos 2 pi u3, r' sin 2 pi u3), u = ((x >> 8) + 0.5) 2^-24,
    r = sqrt(-2 ln u0), r' = sqrt(-2 ln u2)."""
    q, f, b = np.meshgrid(np.arange(win // 4), np.arange(frames), np.arange(B), indexing="ij")
    ctr = np.stack([q, f, b, np.zeros_like(q)], axis=-1).astype(np.uint32)
    w = philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).astype(np.float64)       # (q, f, b, 4)
    u = (np.floor(w / 256.0) + 0.5) * 2.0 ** -24
    out = np.empty(w.shape)
    for a in (0, 2):
        r = np.sqrt(-2.0 * np.log(u[..., a]))
        out[..., a] = r * np.cos(2 * math.pi * u[..., a + 1])
        out[..., a + 1] = r * np.sin(2 * math.pi * u[..., a + 1])
    return out.transpose(2, 1, 0, 3).reshape(B, frames, win)


def fbank(waveform: torch.Tensor, num_mel_bins: int = 80, noise: Optional[torch.Tensor] = None,
          dtype=torch.float32) -> torch.Tensor:
    """O.fbank (25 ms / 10 ms at 16 kHz, povey) with ``noise`` (m, 400) added after framing."""
    if noise is None:
        return O.fbank(waveform, num_mel_bins, dtype=dtype)
    wav = waveform.to(dtype).reshape(-1)
    m = O.num_frames(wav.numel())
    if m == 0:
        return torch.empty(0, num_mel_bins)
    frames = wav.as_strided((m, 400), (160, 1)) + noise.to(dtype)[:m]      # kaldi.py _get_window: + randn * dither
    frames = frames - frames.mean(dim=1, keepdim=True)
    prev = F.pad(frames.unsqueeze(0), (1, 0), mode="replicate").squeeze(0)[:, :-1]
    frames = (frames - 0.97 * prev) * O.povey_window(400, dtype).unsqueeze(0)
    spec = torch.fft.rfft(F.pad(frames, (0, 112))).abs().pow(2.0)
    e = torch.mm(spec, O.mel_banks(num_mel_bins, 512, 16000.0, dtype=dtype).T)
    return torch.max(e, torch.tensor(O.EPS, dtype=dtype)).log()


def mfcc(waveform: torch.Tensor, num_ceps: int = 80, num_mel_bins: int = 80, noise: Optional[torch.Tensor] = None,
         cepstral_lifter: float = 22.0, dtype=torch.float32) -> torch.Tensor:
    """O.mfcc with ``noise`` added after framing."""
    if noise is None:
        return O.mfcc(waveform, num_ceps, num_mel_bins, cepstral_lifter, dtype=dtype)
    f = fbank(waveform, num_mel_bins, noise, dtype)
    if f.shape[0] == 0:
        return torch.empty(0, num_ceps)
    out = f.matmul(O.dct_matrix(num_ceps, num_mel_bins, dtype))
    i = torch.arange(num_ceps)
    return out * (1.0 + 0.5 * cepstral_lifter * torch.sin(math.pi * i / cepstral_lifter)).to(dtype).unsqueeze(0)


def golden_audio() -> Tuple[np.ndarray, List[int]]:
    """The golden's int16 batch: 7 rows of 0.4-0.8 s at 16 kHz (a tone plus noise), one of 15 frames (fewer than the
    recipes' max_t), two of equal length (a tie in padding()'s sort).  Returns (pcm (7, N), lengths)."""
    rng = np.random.default_rng(11)
    lens = [int(v) for v in rng.integers(6400, 12801, 7)]
    lens[2] = 400 + 14 * 160
    lens[5] = lens[1]
    pcm = np.zeros((7, max(lens)), np.int16)
    for b, n in enumerate(lens):
        t = np.arange(n) / 16000.0
        pcm[b, :n] = np.clip(3000 * np.sin(2 * np.pi * (200 + 50 * b) * t) + rng.normal(0, 300, n), -32768, 32767)
    return pcm, lens


def spec_aug_input() -> Tuple[np.ndarray, List[int]]:
    """The golden's SpecAugment input: (5, 120, 40) float32 standard normals and the rows' frame counts."""
    return np.random.default_rng(5).standard_normal((5, 120, 40)).astype(np.float32), [120, 37, 5, 90, 1]


def train_chain(pcm: np.ndarray, lens: Sequence[int], conf: dict, seed: int, rng_seed: int,
                dtype=torch.float64) -> List[torch.Tensor]:
    """Each row through the reference's training chain for ``dataset_conf`` ``conf``, in input order (before
    padding()): features with dither * dither_noise(seed) added after framing, spec_aug with the masks
    random.Random(rng_seed) draws in processor.spec_aug's order, context_expansion, frame_skip."""
    if "feats_type" in conf:
        ftype, fc = conf["feats_type"], conf[conf["feats_type"] + "_conf"]
    else:
        fc = conf["feature_extraction_conf"]
        ftype = fc["feature_type"]
    B = len(lens)
    noise = torch.from_numpy(dither_noise(seed, B, max(O.num_frames(n) for n in lens))) * fc.get("dither", 0.0)
    rng = random.Random(rng_seed)
    out = []
    for b, n in enumerate(lens):
        x = torch.from_numpy(pcm[b, :n].astype(np.float64))
        nz = noise[b, :O.num_frames(n)]
        y = (mfcc(x, fc.get("num_ceps", 80), fc.get("num_mel_bins", 80), nz, dtype=dtype) if ftype == "mfcc"
             else fbank(x, fc.get("num_mel_bins", 23), nz, dtype=dtype))
        if conf.get("spec_aug", True):
            sa = {"num_t_mask": 2, "num_f_mask": 2, "max_t": 50, "max_f": 10, **conf.get("spec_aug_conf", {})}
            y = y.clone()
            for _ in range(sa["num_t_mask"]):
                start = rng.randint(0, y.shape[0] - 1)
                y[start:min(y.shape[0], start + rng.randint(1, sa["max_t"])), :] = 0
            for _ in range(sa["num_f_mask"]):
                start = rng.randint(0, y.shape[1] - 1)
                y[:, start:min(y.shape[1], start + rng.randint(1, sa["max_f"]))] = 0
        if conf.get("context_expansion", False):
            cc = conf.get("context_expansion_conf", {})
            y = O.context_expansion(y, cc.get("left", 1), cc.get("right", 1))
        y = O.frame_skip(y, conf.get("frame_skip", 1))
        out.append(y)
    return out
