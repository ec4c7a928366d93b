"""Global CMVN statistics on the device: the batched twin of the reference's tools/compute_cmvn_stats.py (stage 1 of
every recipe), which loads each utterance, resamples it when ``resample_conf`` asks for it, runs kaldi.fbank or
kaldi.mfcc on it and adds per-dimension sums and sums of squares into accumulators, then writes the ``global_cmvn``
JSON that ``load_cmvn`` / ``init_model(cmvn_file=...)`` read.

Here one ``update`` runs the resampler (csrc/resample.cu, one launch), the Fbank / MFCC kernel (one launch) and the
statistics reduction (csrc/cmvn_stats.cu, two launches) on a batch of utterances at one sample rate.  Two deliberate
differences from the tool:
  * the sums are kept and written in double (the tool keeps float32 accumulators, which on a large set loses
    visible digits of var_stat);
  * feature extraction runs at 16 kHz only: audio at another rate needs ``resample_rate: 16000`` (every shipped
    config sets it), where the tool would run kaldi.fbank at that rate.
"""
from __future__ import annotations

import ctypes as C
import json
from typing import Optional, Sequence, Tuple, Union

import torch

from . import _native
from .frontend import Fbank, Mfcc, Resample

FBANK_RATE = 16000


def scp_segment(value: str, sample_rate: int) -> Tuple[str, Optional[int], Optional[int]]:
    """A wav.scp value as compute_cmvn_stats.py:31-47 reads it: ``path`` or ``path,start_s,end_s``.  Returns
    (path, start, end) sample bounds int(float(t) * sample_rate) of a segment, or (path, None, None)."""
    fields = value.strip().split(",")
    if len(fields) not in (1, 3):
        raise ValueError(f"wav.scp value {value!r} has {len(fields)} comma-separated fields; expected 1 or 3")
    if len(fields) == 1:
        return fields[0], None, None
    return fields[0], int(float(fields[1]) * sample_rate), int(float(fields[2]) * sample_rate)


class CmvnStats:
    """Accumulates the global CMVN statistics of feature type ``feat_type`` ('fbank' or 'mfcc') with ``feat_dim``
    mel bins (and as many cepstra for mfcc) on the device.  ``resample_rate`` 0 = no resampling."""

    def __init__(self, feat_type: str, feat_dim: int, resample_rate: int = 0):
        if feat_type == "fbank":
            self.frontend = Fbank(feat_dim)
        elif feat_type == "mfcc":
            self.frontend = Mfcc(feat_dim, feat_dim)
        else:
            raise ValueError(f"feats_type {feat_type!r}: compute_cmvn_stats handles 'fbank' and 'mfcc'")
        if resample_rate not in (0, FBANK_RATE):
            raise NotImplementedError(f"resample_rate {resample_rate}: the Fbank kernel runs at {FBANK_RATE} Hz only")
        self.feat_type, self.feat_dim, self.resample_rate = feat_type, int(feat_dim), int(resample_rate)
        self._resamplers = {}
        self._acc = None            # (2, D) float64: sum x, sum x^2
        self._frames = None         # (1,) int64

    @classmethod
    def from_config(cls, configs: dict) -> "CmvnStats":
        """The keys compute_cmvn_stats.py:109-116 reads (KeyError on a legacy feature_extraction_conf config)."""
        ds = configs["dataset_conf"]
        feat_type = ds["feats_type"]
        feat_dim = ds[f"{feat_type}_conf"]["num_mel_bins"]
        resample_rate = ds["resample_conf"]["resample_rate"] if "resample_conf" in ds else 0
        return cls(feat_type, feat_dim, resample_rate)

    def _resampler(self, orig: int) -> Resample:
        rs = self._resamplers.get(orig)
        if rs is None:
            rs = self._resamplers[orig] = Resample(orig, self.resample_rate)
        return rs

    def update(self, pcm: torch.Tensor, lengths: Union[Sequence[int], torch.Tensor, None], sample_rate: int) -> None:
        """Adds the utterances of ``pcm`` (B, N) (int16 or float32 at int16 scale, CUDA), row b = its first
        lengths[b] samples, all at ``sample_rate``."""
        if not pcm.is_cuda:
            raise RuntimeError("wekws_b200.CmvnStats runs on CUDA (sm_90a) only; got a CPU tensor (no CPU fallback)")
        if pcm.dim() != 2:
            raise ValueError("pcm must be (B, N)")
        B, N = pcm.shape
        lens = [N] * B if lengths is None else [int(n) for n in (
            lengths.tolist() if isinstance(lengths, torch.Tensor) else lengths)]
        if len(lens) != B or any(n < 0 or n > N for n in lens):
            raise ValueError(f"lengths must be {B} values in 0..{N}")
        dev = pcm.device
        if self._acc is None:
            self._acc = torch.zeros(2, self.feat_dim, dtype=torch.float64, device=dev)
            self._frames = torch.zeros(1, dtype=torch.int64, device=dev)
        elif self._acc.device != dev:
            raise ValueError(f"CmvnStats accumulates on {self._acc.device}; got a batch on {dev}")
        rate = int(sample_rate)
        rs = None
        if self.resample_rate != 0 and self.resample_rate != rate:
            rs = self._resampler(rate)
            rate = self.resample_rate
        if rate != FBANK_RATE:
            raise NotImplementedError(f"audio at {rate} Hz without resample_conf: the Fbank kernel runs at "
                                      f"{FBANK_RATE} Hz only (set dataset_conf.resample_conf.resample_rate: 16000)")
        out_lens = lens if rs is None else [rs.output_length(n) for n in lens]
        for b, n in enumerate(out_lens):
            if n < self.frontend.win:        # kaldi.fbank / kaldi.mfcc assert on a waveform shorter than a frame
                raise ValueError(f"utterance {b} has {n} samples at {FBANK_RATE} Hz, fewer than one "
                                 f"{self.frontend.win}-sample frame")
        if B == 0:
            return
        wave = pcm
        if rs is not None:
            wave = rs(pcm, torch.tensor(lens, dtype=torch.int32).to(dev))
        d_lens = torch.tensor(out_lens, dtype=torch.int32).to(dev)
        d_frames = torch.tensor([self.frontend.num_frames(n) for n in out_lens], dtype=torch.int32).to(dev)
        feats = self.frontend(wave, lengths=d_lens)
        ws = torch.empty(_native.lib().wekws_cmvn_stats_workspace_bytes(B, self.feat_dim), dtype=torch.uint8,
                         device=dev)
        with torch.cuda.device(dev):
            stream = torch.cuda.current_stream(dev).cuda_stream
            rc = _native.lib().wekws_cmvn_stats_accumulate(
                C.c_void_p(feats.data_ptr()), B, feats.shape[1], self.feat_dim, C.c_void_p(d_frames.data_ptr()),
                C.c_void_p(self._acc.data_ptr()), C.c_void_p(self._frames.data_ptr()), C.c_void_p(ws.data_ptr()),
                C.c_void_p(stream))
        _native.check(rc, "wekws_cmvn_stats_accumulate")

    @property
    def frame_num(self) -> int:
        return 0 if self._frames is None else int(self._frames.item())

    @property
    def mean_stat(self) -> torch.Tensor:
        """Per-dimension sum of the features (float64, host)."""
        return torch.zeros(self.feat_dim, dtype=torch.float64) if self._acc is None else self._acc[0].cpu()

    @property
    def var_stat(self) -> torch.Tensor:
        """Per-dimension sum of the squared features (float64, host)."""
        return torch.zeros(self.feat_dim, dtype=torch.float64) if self._acc is None else self._acc[1].cpu()

    def to_json(self) -> str:
        """The tool's schema (compute_cmvn_stats.py:144-151)."""
        acc = torch.zeros(2, self.feat_dim, dtype=torch.float64) if self._acc is None else self._acc.cpu()
        return json.dumps({"mean_stat": acc[0].tolist(), "var_stat": acc[1].tolist(), "frame_num": self.frame_num})

    def write(self, path: str) -> None:
        with open(path, "w") as f:
            f.write(self.to_json())
