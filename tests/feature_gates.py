"""The gates the Fbank / MFCC kernel's features are held to, shared by every test that checks them.

Log-mel: within 1e-3 max-abs / 1e-5 mean-abs of the float32 restatement (SURVEY 8c: the oracle's own fp32-vs-fp64
noise floor is 9e-5..4.3e-4).  MFCC: 6e-3 / 6e-4 (the fp32 restatement sits 3.5e-3 max / 3.5e-4 mean from float64:
sgemm over 80 log-mels of magnitude ~16).  Where the float32 restatement's own rounding exceeds that gate (pure tones:
energy in a few bins, the rest is rounding noise), the kernel must instead be at least as close to the float64
evaluation of the same formulas as the restatement is (x1.5 slack, ``slack``).

``kw`` are the front-end options of ``O.fbank`` / ``O.mfcc`` (window_type, sample_frequency, low_freq, ...), passed
through to the float64 evaluation; ``mean`` / ``istd`` the CMVN the features were normalised with, applied to it in
float64.  Both checks return (max, mean) of |out - ref| so callers can print them."""
import numpy as np
import torch

from oracle import kws_oracle as O

TOL_FEAT_MAX, TOL_FEAT_MEAN = 1e-3, 1e-5
TOL_MFCC_MAX, TOL_MFCC_MEAN = 6e-3, 6e-4


def _cmvn64(x, mean, istd):
    if mean is not None:
        x = x - mean.double()
    if istd is not None:
        x = x * istd.double()
    return x


def _check(out, ref, what, tmax, tmean, truth, slack):
    assert out.shape == ref.shape, what
    if not ref.size:
        return 0.0, 0.0
    d = np.abs(out - ref)
    if d.max() <= tmax and d.mean() <= tmean:
        return float(d.max()), float(d.mean())
    assert truth is not None, (what, d.max(), d.mean())
    t = truth().numpy()
    e_ref, e_out = np.abs(ref - t), np.abs(out - t)
    assert e_out.max() <= max(tmax, slack * e_ref.max()), (what, e_out.max(), e_ref.max())
    assert e_out.mean() <= max(tmean, slack * e_ref.mean()), (what, e_out.mean(), e_ref.mean())
    return float(d.max()), float(d.mean())


def check_feats(out, ref, what, wav=None, mean=None, istd=None, slack=1.5, **kw):
    """Log-mel ``out`` (m, nmel) against ``ref``, the float32 restatement of the same features (or the reference's
    own output); the float64 fallback needs ``wav``, the waveform both were computed from."""
    truth = None if wav is None else lambda: _cmvn64(O.fbank(wav, dtype=torch.float64, **kw), mean, istd)
    return _check(out, ref, what, TOL_FEAT_MAX, TOL_FEAT_MEAN, truth, slack)


def check_mfcc(out, ref, what, wav, nc, nmel, mean=None, istd=None, slack=1.5, **kw):
    """MFCC ``out`` (m, nc) against ``ref`` as check_feats; ``kw`` may include cepstral_lifter."""
    truth = lambda: _cmvn64(O.mfcc(wav, nc, nmel, dtype=torch.float64, **kw), mean, istd)   # noqa: E731
    return _check(out, ref, what, TOL_MFCC_MAX, TOL_MFCC_MEAN, truth, slack)
