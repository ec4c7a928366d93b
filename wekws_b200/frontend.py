"""Kaldi-compatible log-mel filterbank front-end on the GPU.

Drop-in for the one call the reference makes into torchaudio,
``kaldi.fbank(waveform, num_mel_bins=..., frame_length=25, frame_shift=10, dither=0.0,
energy_floor=0.0, sample_frequency=16000)`` (wekws/dataset/processor.py:196-202,
wekws/bin/stream_kws_ctc.py:354-360), extended to batches of waveforms and optionally fused
with global CMVN (wekws/model/cmvn.py:45-47).  Host code here only prepares the constants
(window, mel weights) with the same fp32 torch ops torchaudio uses, so the tables are
bit-identical to the reference's; the computation is the sm_90a kernel in csrc/fbank.cu.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import numpy as np
import torch

from . import _native

EPSILON = float(torch.finfo(torch.float32).eps)      # torchaudio kaldi.py:21


def window_function(window_type: str, n: int) -> torch.Tensor:
    """torchaudio kaldi.py:88-110 (povey default; hamming matches runtime/core/frontend/fbank.h:90-96)."""
    if window_type == "povey":
        return torch.hann_window(n, periodic=False, dtype=torch.float32).pow(0.85)
    if window_type == "hanning":
        return torch.hann_window(n, periodic=False, dtype=torch.float32)
    if window_type == "hamming":
        return torch.hamming_window(n, periodic=False, alpha=0.54, beta=0.46, dtype=torch.float32)
    if window_type == "rectangular":
        return torch.ones(n, dtype=torch.float32)
    raise ValueError("Invalid window type " + window_type)


def mel_filterbank(num_bins: int, n_fft: int, sample_freq: float, low_freq: float = 20.0,
                   high_freq: float = 0.0) -> torch.Tensor:
    """(num_bins, n_fft // 2) triangular weights, torchaudio kaldi.py:436-511 (no VTLN)."""
    assert num_bins > 3, "Must have at least 3 mel bins"
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    assert 0.0 <= low_freq < nyquist and 0.0 < high_freq <= nyquist and low_freq < high_freq
    bin_width = sample_freq / n_fft
    lo = 1127.0 * math.log(1.0 + low_freq / 700.0)
    hi = 1127.0 * math.log(1.0 + high_freq / 700.0)
    step = (hi - lo) / (num_bins + 1)
    idx = torch.arange(num_bins).unsqueeze(1)
    left, center, right = lo + idx * step, lo + (idx + 1.0) * step, lo + (idx + 2.0) * step
    mel = (1127.0 * (1.0 + (bin_width * torch.arange(n_fft // 2, dtype=torch.float32)) / 700.0).log()).unsqueeze(0)
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    return torch.max(torch.zeros(1), torch.min(up, down)).contiguous()


def dct_matrix(num_ceps: int, num_mel_bins: int) -> torch.Tensor:
    """(num_mel_bins, num_ceps) DCT-II matrix of torchaudio kaldi.py `_get_dct_matrix`: ortho-normalised
    create_dct(n, n, 'ortho') with the first column replaced by sqrt(1/n), truncated to num_ceps columns."""
    n = torch.arange(float(num_mel_bins))
    k = torch.arange(float(num_mel_bins)).unsqueeze(1)
    dct = torch.cos(math.pi / float(num_mel_bins) * (n + 0.5) * k)      # (n_mfcc, n_mels)
    dct[0] *= 1.0 / math.sqrt(2.0)
    dct *= math.sqrt(2.0 / float(num_mel_bins))
    dct = dct.t().contiguous()
    dct[:, 0] = math.sqrt(1 / float(num_mel_bins))
    return dct[:, :num_ceps].contiguous()


def lifter_coeffs(num_ceps: int, cepstral_lifter: float) -> torch.Tensor:
    """torchaudio kaldi.py `_get_lifter_coeffs`: 1 + 0.5 Q sin(pi i / Q)."""
    i = torch.arange(num_ceps)
    return 1.0 + 0.5 * cepstral_lifter * torch.sin(math.pi * i / cepstral_lifter)


class Fbank:
    """Batched GPU Fbank(+CMVN).  ``__call__(pcm)``: pcm (B, N) or (N,) int16 / float32 CUDA
    tensor in int16 scale (the reference multiplies normalised audio by 1<<15 first,
    processor.py:194) -> (B, m, num_mel_bins) float32 with m = 1 + (N - 400) // 160."""

    def __init__(self, num_mel_bins: int = 80, frame_length: float = 25.0, frame_shift: float = 10.0,
                 sample_frequency: float = 16000.0, window_type: str = "povey",
                 preemphasis_coefficient: float = 0.97, remove_dc_offset: bool = True,
                 low_freq: float = 20.0, high_freq: float = 0.0, device: Optional[torch.device] = None):
        self.num_mel_bins = num_mel_bins
        self.win = int(sample_frequency * frame_length * 0.001)
        self.shift = int(sample_frequency * frame_shift * 0.001)
        self.n_fft = 1 if self.win == 0 else 2 ** (self.win - 1).bit_length()
        self.cfg = _native.FbankConfig(int(sample_frequency), self.win, self.shift, self.n_fft, num_mel_bins,
                                       float(preemphasis_coefficient), int(bool(remove_dc_offset)), EPSILON)
        self.window = window_function(window_type, self.win).contiguous()
        self.mel = mel_filterbank(num_mel_bins, self.n_fft, sample_frequency, low_freq, high_freq)
        self._handles = {}
        self.device = device
        self.feature_dim = num_mel_bins          # row width of the output (num_ceps for the Mfcc subclass)

    def _configure(self, handle) -> None:
        """Hook for subclasses: extra native configuration of a freshly created handle."""

    def num_frames(self, num_samples: int) -> int:
        return 0 if num_samples < self.win else 1 + (num_samples - self.win) // self.shift

    def _handle(self, dev: torch.device):
        h = self._handles.get(dev)
        if h is None:
            h = C.c_void_p()
            with torch.cuda.device(dev):
                _native.check(_native.lib().wekws_fbank_create(
                    C.byref(self.cfg), C.c_void_p(self.window.data_ptr()), C.c_void_p(self.mel.data_ptr()),
                    C.byref(h)), "wekws_fbank_create")
                self._configure(h)
            self._handles[dev] = h
        return h

    def __del__(self):
        for h in getattr(self, "_handles", {}).values():
            try:
                _native.lib().wekws_fbank_destroy(h)
            except Exception:
                pass

    def __call__(self, pcm: torch.Tensor, lengths: Optional[torch.Tensor] = None,
                 mean: Optional[torch.Tensor] = None, istd: Optional[torch.Tensor] = None,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
        if not pcm.is_cuda:
            raise RuntimeError("wekws_b200.Fbank runs on CUDA (sm_90a) only; got a CPU tensor (no CPU fallback)")
        squeeze = pcm.dim() == 1
        if squeeze:
            pcm = pcm.unsqueeze(0)
        if pcm.dim() != 2:
            raise ValueError("pcm must be (N,) or (B, N)")
        if pcm.dtype == torch.int16:
            dtype = _native.PCM_S16
        elif pcm.dtype == torch.float32:
            dtype = _native.PCM_F32
        else:
            raise TypeError(f"pcm must be int16 or float32, got {pcm.dtype}")
        if pcm.stride(1) != 1:
            pcm = pcm.contiguous()
        dev = pcm.device
        B, N = pcm.shape
        m = self.num_frames(N)
        if out is None:
            out = torch.empty(B, m, self.feature_dim, device=dev, dtype=torch.float32)
        elif tuple(out.shape) != (B, m, self.feature_dim) or not out.is_contiguous():
            raise ValueError("out must be a contiguous (B, m, feature_dim) tensor")

        def ptr(t, dt):
            if t is None:
                return None
            t = t.to(device=dev, dtype=dt).contiguous()
            keep.append(t)
            return C.c_void_p(t.data_ptr())

        keep = []
        if B > 0 and m > 0:
            h = self._handle(dev)
            with torch.cuda.device(dev):
                stream = torch.cuda.current_stream(dev).cuda_stream
                rc = _native.lib().wekws_fbank_forward(
                    h, C.c_void_p(pcm.data_ptr()), dtype, B, N, pcm.stride(0), ptr(lengths, torch.int32),
                    ptr(mean, torch.float32), ptr(istd, torch.float32), C.c_void_p(out.data_ptr()), m,
                    C.c_void_p(stream))
            _native.check(rc, "wekws_fbank_forward")
        return out[0] if squeeze else out


class Mfcc(Fbank):
    """Batched GPU MFCC(+CMVN): the Fbank kernel with a fused DCT-II + lifter epilogue.  Mirrors
    ``kaldi.mfcc(waveform, num_ceps=..., num_mel_bins=..., frame_length=25, frame_shift=10, dither=0.0,
    energy_floor=0.0, sample_frequency=...)`` (wekws/dataset/processor.py:157-166; the front-end of the shipped
    mdtc configs, examples/hi_xiaowen/s0/conf/mdtc.yaml:8-14) -> (B, m, num_ceps).  mean / istd passed to
    ``__call__`` are applied to the cepstra."""

    def __init__(self, num_ceps: int = 80, num_mel_bins: int = 80, cepstral_lifter: float = 22.0, **kw):
        if num_ceps > num_mel_bins:
            raise AssertionError("num_ceps cannot be larger than num_mel_bins: %d vs %d" % (num_ceps, num_mel_bins))
        super().__init__(num_mel_bins, **kw)
        self.num_ceps = num_ceps
        self.feature_dim = num_ceps
        self.dct = dct_matrix(num_ceps, num_mel_bins)
        self.lifter = lifter_coeffs(num_ceps, cepstral_lifter).float().contiguous() if cepstral_lifter != 0.0 else None

    def _configure(self, handle) -> None:
        _native.check(_native.lib().wekws_fbank_set_mfcc(
            handle, self.num_ceps, C.c_void_p(self.dct.data_ptr()),
            C.c_void_p(self.lifter.data_ptr()) if self.lifter is not None else None), "wekws_fbank_set_mfcc")


def sinc_resample_kernel(orig_freq: int, new_freq: int, lowpass_filter_width: int = 6, rolloff: float = 0.99,
                         resampling_method: str = "sinc_interp_hann"):
    """torchaudio 2.11 functional `_get_sinc_resample_kernel` with dtype None: the same float64 ops in the same order,
    then a cast to float32.  Returns the (new / g, 2 width + orig / g) table and width (g = gcd of the rates).
    Only the Hann window is implemented: it is the only one the reference uses."""
    if resampling_method != "sinc_interp_hann":
        raise NotImplementedError(f"resampling_method {resampling_method!r}: only 'sinc_interp_hann' is implemented")
    if int(orig_freq) != orig_freq or int(new_freq) != new_freq:
        raise ValueError("resample rates must be integers")
    if lowpass_filter_width <= 0:
        raise ValueError("Low pass filter width should be positive.")
    g = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // g, int(new_freq) // g
    base_freq = min(orig, new) * rolloff
    width = math.ceil(lowpass_filter_width * orig / base_freq)
    if new * (2 * width + orig) > _RESAMPLE_DENSE_MAX:
        raise ValueError(f"resample {orig_freq} -> {new_freq}: the filter table is {new} x {2 * width + orig} floats; "
                         f"its non-zero taps (about {new * math.ceil(2 * lowpass_filter_width * orig / base_freq) * 4} "
                         "bytes) do not fit the kernel's shared memory")
    idx = torch.arange(-width, width + orig, dtype=torch.float64)[None, None] / orig
    t = torch.arange(0, -new, -1, dtype=None)[:, None, None] / new + idx
    t *= base_freq
    t = t.clamp_(-lowpass_filter_width, lowpass_filter_width)
    window = torch.cos(t * math.pi / lowpass_filter_width / 2) ** 2
    t *= math.pi
    scale = base_freq / orig
    kernels = torch.where(t == 0, torch.tensor(1.0).to(t), t.sin() / t)
    kernels *= window * scale
    return kernels.to(dtype=torch.float32), width


_RESAMPLE_DENSE_MAX = 1 << 24        # dense table entries; far past any pair whose compact table fits on chip


class Resample:
    """Batched GPU twin of ``torchaudio.transforms.Resample(orig_freq, new_freq)`` (sinc_interp_hann,
    lowpass_filter_width 6, rolloff 0.99), as wekws/dataset/processor.py resample() and tools/compute_cmvn_stats.py
    call it.  ``__call__(pcm, lengths=None)``: pcm (B, N) or (N,) int16 / float32 CUDA tensor at int16 scale ->
    (B, output_length(N)) float32; row b is the resampling of its first lengths[b] samples (the rest count as zeros
    and are never read), zero-filled past output_length(lengths[b]).  The output is not rounded back to int16:
    kaldi.fbank receives the float waveform.  Each output is accumulated in double and rounded once to float32."""

    def __init__(self, orig_freq: int, new_freq: int, resampling_method: str = "sinc_interp_hann",
                 lowpass_filter_width: int = 6, rolloff: float = 0.99):
        self.orig_freq, self.new_freq = int(orig_freq), int(new_freq)
        if self.orig_freq <= 0 or self.new_freq <= 0:
            raise ValueError(f"resample rates must be positive, got {orig_freq} -> {new_freq}")
        self.gcd = math.gcd(self.orig_freq, self.new_freq)
        self.kernel, self.width = None, 0
        if self.orig_freq != self.new_freq:
            self.kernel, self.width = sinc_resample_kernel(self.orig_freq, self.new_freq, lowpass_filter_width,
                                                           rolloff, resampling_method)
            self.kernel = self.kernel.reshape(self.kernel.shape[0], -1).contiguous()
        self._handles = {}

    def output_length(self, num_samples: int) -> int:
        """torchaudio's target length ceil(torch.as_tensor(new * n / orig)): the quotient passes through float32, so
        for very long rows it can be one short of the exact ceiling; n itself when the rates are equal."""
        if self.orig_freq == self.new_freq:
            return int(num_samples)
        o, n = self.orig_freq // self.gcd, self.new_freq // self.gcd
        if num_samples <= 0:
            return 0
        target = math.ceil(float(np.float32(n * int(num_samples) / o)))
        return min(target, (int(num_samples) // o + 1) * n)

    def _handle(self, dev: torch.device):
        h = self._handles.get(dev)
        if h is None:
            h = C.c_void_p()
            with torch.cuda.device(dev):
                _native.check(_native.lib().wekws_resample_create(
                    self.orig_freq, self.new_freq, C.c_void_p(self.kernel.data_ptr()), self.width, C.byref(h)),
                    "wekws_resample_create")
            self._handles[dev] = h
        return h

    def __del__(self):
        for h in getattr(self, "_handles", {}).values():
            try:
                _native.lib().wekws_resample_destroy(h)
            except Exception:
                pass

    def __call__(self, pcm: torch.Tensor, lengths=None) -> torch.Tensor:
        if self.orig_freq == self.new_freq:
            return pcm                       # as the transform does
        if not pcm.is_cuda:
            raise RuntimeError("wekws_b200.Resample runs on CUDA (sm_90a) only; got a CPU tensor (no CPU fallback)")
        squeeze = pcm.dim() == 1
        if squeeze:
            pcm = pcm.unsqueeze(0)
        if pcm.dim() != 2:
            raise ValueError("pcm must be (N,) or (B, N)")
        if pcm.dtype == torch.int16:
            dtype = _native.PCM_S16
        elif pcm.dtype == torch.float32:
            dtype = _native.PCM_F32
        else:
            raise TypeError(f"pcm must be int16 or float32, got {pcm.dtype}")
        if pcm.stride(1) != 1:
            pcm = pcm.contiguous()
        dev = pcm.device
        B, N = pcm.shape
        max_out = self.output_length(N)
        out = torch.empty(B, max_out, device=dev, dtype=torch.float32)
        lens = None
        if lengths is not None:
            lens = torch.as_tensor(lengths).to(device=dev, dtype=torch.int32).contiguous()
            if lens.shape != (B,):
                raise ValueError(f"lengths must have shape ({B},), got {tuple(lens.shape)}")
        if B > 0 and max_out > 0:
            h = self._handle(dev)
            with torch.cuda.device(dev):
                stream = torch.cuda.current_stream(dev).cuda_stream
                rc = _native.lib().wekws_resample_forward(
                    h, C.c_void_p(pcm.data_ptr()), dtype, B, N, pcm.stride(0),
                    C.c_void_p(lens.data_ptr()) if lens is not None else None, C.c_void_p(out.data_ptr()),
                    out.stride(0), max_out, C.c_void_p(stream))
            _native.check(rc, "wekws_resample_forward")
        return out[0] if squeeze else out


def resample(waveform: torch.Tensor, orig_freq: int, new_freq: int) -> torch.Tensor:
    """Functional form: the waveform unchanged when the rates are equal (as the transform does), else
    Resample(orig_freq, new_freq)(waveform) with the handle cached per rate pair."""
    key = ("resample", int(orig_freq), int(new_freq))
    rs = _DEFAULT.get(key)
    if rs is None:
        rs = _DEFAULT[key] = Resample(orig_freq, new_freq)
    return rs(waveform)


_DEFAULT = {}


def fbank(waveform: torch.Tensor, num_mel_bins: int = 23, frame_length: float = 25.0,
          frame_shift: float = 10.0, dither: float = 0.0, energy_floor: float = 0.0,
          sample_frequency: float = 16000.0, window_type: str = "povey") -> torch.Tensor:
    """Signature-compatible subset of torchaudio.compliance.kaldi.fbank for the reference's
    call sites: waveform (1, N) -> (m, num_mel_bins).  dither must be 0 (test-time setting)."""
    if dither != 0.0:
        raise NotImplementedError("wekws_b200.fbank: dither is a training-time augmentation; use dither=0.0")
    key = (num_mel_bins, frame_length, frame_shift, sample_frequency, window_type)
    fb = _DEFAULT.get(key)
    if fb is None:
        fb = _DEFAULT[key] = Fbank(num_mel_bins, frame_length, frame_shift, sample_frequency, window_type)
    if waveform.dim() == 2:
        assert waveform.size(0) == 1, "kaldi.fbank expects a mono (1, N) waveform"
        return fb(waveform)[0]
    return fb(waveform)


def mfcc(waveform: torch.Tensor, num_ceps: int = 13, num_mel_bins: int = 23, frame_length: float = 25.0,
         frame_shift: float = 10.0, dither: float = 0.0, energy_floor: float = 0.0,
         sample_frequency: float = 16000.0, cepstral_lifter: float = 22.0, window_type: str = "povey") -> torch.Tensor:
    """Signature-compatible subset of torchaudio.compliance.kaldi.mfcc for the reference's call site
    (processor.py:157-166): waveform (1, N) -> (m, num_ceps).  dither must be 0 (test-time setting)."""
    if dither != 0.0:
        raise NotImplementedError("wekws_b200.mfcc: dither is a training-time augmentation; use dither=0.0")
    key = ("mfcc", num_ceps, num_mel_bins, frame_length, frame_shift, sample_frequency, cepstral_lifter, window_type)
    fe = _DEFAULT.get(key)
    if fe is None:
        fe = _DEFAULT[key] = Mfcc(num_ceps, num_mel_bins, cepstral_lifter, frame_length=frame_length,
                                  frame_shift=frame_shift, sample_frequency=sample_frequency, window_type=window_type)
    if waveform.dim() == 2:
        assert waveform.size(0) == 1, "kaldi.mfcc expects a mono (1, N) waveform"
        return fe(waveform)[0]
    return fe(waveform)
