"""CPU oracle of the training-audio augmentation (wekws_b200/augment.py, csrc/augment.cu).  TEST INFRASTRUCTURE ONLY.

* ``reverb_f64``: processor.add_reverb's arithmetic in float64, convolve(x, rir / sqrt(sum rir^2), 'full')[:n] as a
  direct sum;
* ``noise_f64`` / ``noise_f32``: processor.add_noise's arithmetic at int16 scale: the gain in float64 (audio level at
  the reference's [-1, 1] scale, hence the 2^-15), then x + gain s in float64, or with the device's two float32
  roundings;
* ``noise_segment``: the segment a row adds (a slice of a longer clip, np.resize's repetition of a shorter one);
* ``audio`` / ``rir_items`` / ``noise_items``: the seeded inputs of tests/golden/augment.npz, which stores only the
  reference's outputs and the ``random`` calls it made (oracle/make_augment_golden.py);
* ``Recorder``: a ``random`` stand-in that logs every call, to compare draw sequences.
"""
from __future__ import annotations

import io
import json
import random
from typing import List, Optional, Sequence, Tuple

import numpy as np


def wav_bytes(a: np.ndarray, rate: int = 16000) -> bytes:
    from scipy.io import wavfile
    f = io.BytesIO()
    wavfile.write(f, rate, a)
    return f.getvalue()


def _decay(rng, n: int, scale: float, tau: float) -> np.ndarray:
    return rng.standard_normal(n) * scale * np.exp(-np.arange(n) / tau)


def audio() -> Tuple[np.ndarray, List[int]]:
    """The golden's int16 batch: 10 rows of 0.1-0.6 s at 16 kHz, noise shaped by a slow random envelope (speech-like
    levels, no pure tones); row 3 is 8000 samples, the length of one noise clip.  Returns (pcm (10, N), lengths)."""
    rng = np.random.default_rng(21)
    lens = [int(v) for v in rng.integers(1600, 9601, 10)]
    lens[3] = 8000
    pcm = np.zeros((10, max(lens)), np.int16)
    for b, n in enumerate(lens):
        env = np.interp(np.arange(n), np.linspace(0, n, 9), rng.uniform(0.05, 1.0, 9))
        x = np.convolve(rng.standard_normal(n + 15), np.hanning(16) / 4, "valid")[:n]
        pcm[b, :n] = np.clip(np.round(4000 * env * x), -32768, 32767)
    return pcm, lens


def rir_items() -> List[Tuple[str, bytes]]:
    """RIRs of 1, 31, 4000 (float32 WAV), 16000 (longer than every row) and a stereo 3000-tap one."""
    rng = np.random.default_rng(22)
    i16 = lambda a: np.clip(np.round(a), -32768, 32767).astype(np.int16)      # noqa: E731
    stereo = np.stack([i16(_decay(rng, 3000, 9000, 500)), i16(_decay(rng, 3000, 9000, 300))], axis=1)
    return [("rir_1", wav_bytes(np.array([12000], np.int16))),
            ("rir_31", wav_bytes(i16(_decay(rng, 31, 8000, 8)))),
            ("rir_4000", wav_bytes(_decay(rng, 4000, 0.5, 700).astype(np.float32))),
            ("rir_16000", wav_bytes(i16(_decay(rng, 16000, 10000, 2500)))),
            ("rir_stereo", wav_bytes(stereo))]


def noise_items() -> List[Tuple[str, bytes]]:
    """Noise clips of the four key prefixes: shorter than every row (1200), equal to row 3 (8000) and longer than
    every row (20000); int16 and float32 WAVs."""
    rng = np.random.default_rng(23)
    i16 = lambda a: np.clip(np.round(a), -32768, 32767).astype(np.int16)      # noqa: E731
    return [("noise_short", wav_bytes(i16(rng.standard_normal(1200) * 3000))),
            ("speech_equal", wav_bytes((rng.standard_normal(8000) * 0.2).astype(np.float32))),
            ("music_long", wav_bytes(i16(rng.standard_normal(20000) * 5000))),
            ("babble_long", wav_bytes(i16(rng.standard_normal(20000) * 800))),
            ("noise_long_f32", wav_bytes((rng.standard_normal(20000) * 1500).astype(np.float32)))]


def decode(data: bytes) -> np.ndarray:
    from scipy.io import wavfile
    a = wavfile.read(io.BytesIO(data))[1].astype(np.float32)
    return a[:, 0] if a.ndim > 1 else a


def reverb_f64(x: np.ndarray, rir: np.ndarray) -> np.ndarray:
    """convolve(x, h, 'full')[:len(x)] with h = rir / sqrt(sum rir^2), all in float64 (a direct sum)."""
    r = np.asarray(rir, np.float64)
    h = r / np.sqrt(np.sum(r * r))
    n = len(x)
    return np.convolve(np.asarray(x, np.float64), h[:n])[:n]


def noise_segment(clip: np.ndarray, n: int, start: Optional[int]) -> np.ndarray:
    return clip[start:start + n] if start is not None else np.resize(clip, (n,))


def noise_gain(x: np.ndarray, s: np.ndarray, snr: float) -> float:
    """2^15 sqrt(10^((audio_db - noise_db - snr) / 10)) in float64, x at int16 scale, s the segment."""
    a = np.asarray(x, np.float64) * 2.0 ** -15
    audio_db = 10 * np.log10(np.mean(a * a) + 1e-4)
    noise_db = 10 * np.log10(np.mean(np.asarray(s, np.float64) ** 2) + 1e-4)
    return 32768.0 * float(np.sqrt(10 ** ((audio_db - noise_db - snr) / 10)))


def noise_f64(x: np.ndarray, s: np.ndarray, snr: float) -> np.ndarray:
    return np.asarray(x, np.float64) + noise_gain(x, s, snr) * np.asarray(s, np.float64)


def noise_f32(x: np.ndarray, s: np.ndarray, snr: float) -> np.ndarray:
    g = np.float32(noise_gain(x, s, snr))
    return (np.asarray(x, np.float32) + (g * np.asarray(s, np.float32)).astype(np.float32)).astype(np.float32)


def snr_range(key: str) -> Tuple[int, int]:
    for prefix, r in (("noise", (0, 15)), ("speech", (5, 30)), ("music", (5, 15))):
        if key.startswith(prefix):
            return r
    return (0, 15)


class Recorder:
    """A ``random`` module stand-in over random.Random(seed) that logs (name, args, result) of every call."""

    def __init__(self, seed):
        self._r = random.Random(seed)
        self.log: list = []

    def _call(self, name, *args):
        v = getattr(self._r, name)(*args)
        self.log.append([name, list(args), v])
        return v

    def random(self):
        return self._call("random")

    def randint(self, a, b):
        return self._call("randint", a, b)

    def uniform(self, a, b):
        return self._call("uniform", a, b)

    def dumps(self) -> str:
        return json.dumps(self.log)


def replay(log_json: str, n_rows: Sequence[int], items, kind: str):
    """The per-row choices a recorded add_reverb (kind 'reverb') or add_noise ('noise') pass made, read back from its
    log: reverb -> B clip indices or None; noise -> B (index, start or None, snr) or None."""
    log = json.loads(log_json)
    lengths = [len(decode(b)) for _, b in items]
    out, p = [], 0
    for n in n_rows:
        assert log[p][0] == "random"
        # the stage's probability is not in the log: a row is selected iff the next call is its clip draw
        p += 1
        if p < len(log) and log[p][0] == "randint" and log[p][1] == [0, len(items) - 1]:
            i = log[p][2]
            p += 1
            if kind == "reverb":
                out.append(i)
                continue
            start = None
            if lengths[i] > n:
                start = log[p][2]
                p += 1
            out.append((i, start, log[p][2]))
            p += 1
        else:
            out.append(None)
    assert p == len(log)
    return out
