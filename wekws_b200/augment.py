"""Training-audio augmentation on the device: the add_reverb / add_noise stages of the legacy training chain
(wekws/dataset/dataset.py Dataset(): resample -> add_reverb -> add_noise -> compute_fbank ...).

The reference draws an RIR, or a noise / speech / music clip, from an LMDB source for each selected utterance and
works on it with numpy / scipy in a data-loader worker.  Here the draws stay on the host, made with Python's
``random`` in processor.add_reverb / add_noise's order, so the same random state selects the same rows, clips, noise
offsets and SNRs.  Only the selected clips (and, for noise, only the segment each row uses) travel to the device, in
one asynchronous copy from pinned memory, and csrc/augment.cu does the arithmetic:
  * ``reverb``: convolve(x, rir / sqrt(sum rir^2), 'full')[:n] with FP64 FMAs, each output within 1 ulp of the
    float64 evaluation (the reference uses scipy's float32 FFT);
  * ``add_noise``: x + gain * s at the reference's SNR, with the decibel levels summed in double.
Deliberate differences from the reference:
  * an all-zero (or empty) RIR is refused when the source is built; the reference would divide by zero and train on
    NaNs.  An empty noise clip is refused too;
  * the RIR's sample rate is ignored, as the reference ignores it.
"""
from __future__ import annotations

import io
import random
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _native

SNR_RANGES = (("noise", (0, 15)), ("speech", (5, 30)), ("music", (5, 15)))
DEFAULT_SNR_RANGE = (0, 15)


def decode_wav(data: bytes) -> np.ndarray:
    """A clip as processor.add_reverb / add_noise decode it: scipy.io.wavfile.read, astype(float32), the first channel
    of a multi-channel file."""
    from scipy.io import wavfile
    _, a = wavfile.read(io.BytesIO(data))
    a = a.astype(np.float32)
    if a.ndim > 1:
        a = a[:, 0]
    return np.ascontiguousarray(a)


def snr_range(key: str) -> Tuple[int, int]:
    """processor.add_noise's SNR range for a noise key: by its prefix noise / speech / music, else (0, 15)."""
    for prefix, rng in SNR_RANGES:
        if key.startswith(prefix):
            return rng
    return DEFAULT_SNR_RANGE


def _lookup(db, key: str) -> bytes:
    if hasattr(db, "get"):
        return db.get(key)
    if hasattr(db, "db"):                          # the reference's LmdbData: an lmdb environment
        with db.db.begin(write=False) as txn:
            return txn.get(key.encode())
    return db[key]


class AugmentSource:
    """A bank of (key, clip) items: the reverb or noise source of the training chain, decoded once on the host.

    ``items``: (key, wav bytes) pairs (or a dict of them), or an object with the reference LmdbData's ``keys`` list
    and a byte look-up (``get(key)``, LmdbData's ``db`` environment, or ``[key]``).  The key order is kept: a draw picks
    ``keys[randint(0, len(keys) - 1)]`` as LmdbData.random_one does.  ``rir=True`` marks an RIR bank: an empty or
    all-zero RIR raises ValueError (the reference would produce NaNs).  Clips are float32 numpy arrays at the scale
    ``wavfile.read(...).astype(float32)`` gives; their lengths stay on the host for the draws."""

    def __init__(self, items, rir: bool = False):
        if isinstance(items, dict):
            pairs = list(items.items())
        elif hasattr(items, "keys") and not callable(items.keys):
            pairs = [(k, _lookup(items, k)) for k in items.keys]
        else:
            pairs = list(items)
        if not pairs:
            raise ValueError("an augmentation source needs at least one clip")
        self.rir = bool(rir)
        self.keys: List[str] = []
        self.clips: List[np.ndarray] = []
        for key, data in pairs:
            if data is None:
                raise KeyError(f"augmentation source: no data for key {key!r}")
            clip = decode_wav(bytes(data))
            if clip.size == 0:
                raise ValueError(f"augmentation source: clip {key!r} is empty")
            if self.rir and not np.any(clip):
                raise ValueError(f"RIR {key!r} is all zeros: it cannot be normalised (the reference would produce "
                                 "NaNs)")
            self.keys.append(str(key))
            self.clips.append(clip)
        self.lengths = [int(c.size) for c in self.clips]

    @classmethod
    def from_lmdb(cls, path: str, rir: bool = False) -> "AugmentSource":
        """Reads an LMDB file in the reference's layout (tools/make_lmdb.py: a pickled key list under b'__keys__',
        each key's wav bytes under the key)."""
        try:
            import lmdb
        except ImportError as e:
            raise ImportError("AugmentSource.from_lmdb needs the `lmdb` package (pip install lmdb); or build the "
                              "source from (key, wav bytes) pairs") from e
        import pickle
        env = lmdb.open(path, readonly=True, lock=False, readahead=False)
        try:
            with env.begin(write=False) as txn:
                obj = txn.get(b"__keys__")
                if obj is None:
                    raise ValueError(f"{path}: no __keys__ entry")
                keys = pickle.loads(obj)
                pairs = [(k, txn.get(k.encode())) for k in keys]
        finally:
            env.close()
        return cls(pairs, rir=rir)

    def __len__(self) -> int:
        return len(self.keys)


def draw_reverb(n: int, source: AugmentSource, prob: float, rng=random, row: int = 0) -> Optional[int]:
    """processor.add_reverb's draws for one utterance of n samples: rng.random(), then on selection the clip index
    (LmdbData.random_one's randint).  Returns the index or None.  A selected empty row raises ValueError, as
    scipy.signal.convolve does."""
    if not prob > rng.random():
        return None
    i = rng.randint(0, len(source.keys) - 1)
    if n <= 0:
        raise ValueError(f"add_reverb: row {row} is empty (scipy.signal.convolve refuses an empty input)")
    return i


def draw_noise(n: int, source: AugmentSource, prob: float, rng=random) -> Optional[Tuple[int, Optional[int], float]]:
    """processor.add_noise's draws for one utterance of n samples: rng.random(); on selection the clip index, the
    segment start randint(0, len - n) only when the clip is longer than the utterance, then the SNR uniform over the
    key's range.  Returns (index, start or None, snr) or None."""
    if not prob > rng.random():
        return None
    i = rng.randint(0, len(source.keys) - 1)
    length = source.lengths[i]
    start = rng.randint(0, length - n) if length > n else None
    lo, hi = snr_range(source.keys[i])
    return i, start, rng.uniform(lo, hi)


def _check(pcm: torch.Tensor, lengths, what: str) -> Tuple[torch.Tensor, List[int]]:
    pcm, _, _ = _native.pcm_rows(pcm, what, one_d=False)
    return pcm, _native.host_lengths(lengths, *pcm.shape)


def _upload(dev, rows: Sequence[int], clips: Sequence[np.ndarray], snr: Optional[Sequence[float]] = None):
    """One pinned host buffer -> one asynchronous copy: [snr doubles][rows int32][clip floats].  Returns the device
    buffer and the byte offsets of the three parts."""
    nf = sum(int(c.size) for c in clips)
    if nf >= 1 << 31:
        raise ValueError(f"{nf} clip samples in one batch: more than the 2^31 a launch addresses")
    ns = 0 if snr is None else len(snr)
    o_rows = 8 * ns
    o_clip = o_rows + 4 * len(rows)
    buf = torch.empty(o_clip + 4 * nf, dtype=torch.uint8, pin_memory=True)
    host = buf.numpy()
    if ns:
        host[:o_rows].view(np.float64)[:] = snr
    host[o_rows:o_clip].view(np.int32)[:] = rows
    flat = host[o_clip:].view(np.float32)
    p = 0
    for c in clips:
        flat[p:p + c.size] = c
        p += c.size
    with torch.cuda.device(dev):
        d = buf.to(dev, non_blocking=True)
    return d, o_rows, o_clip


def launch_reverb(pcm: torch.Tensor, lens: Sequence[int], picks: Sequence[Optional[int]],
                  source: AugmentSource) -> torch.Tensor:
    """The device half of ``reverb``: row b convolved with source clip picks[b] (None = a copy).  pcm (B, N)
    contiguous rows; returns a new float32 (B, N) tensor."""
    pcm, code, _ = _native.pcm_rows(pcm, "reverb", one_d=False)
    B, N = pcm.shape
    dev = pcm.device
    out = torch.empty(B, N, dtype=torch.float32, device=dev)
    offsets, clips, rows, nf = {}, [], [], 0
    for b, i in enumerate(picks):
        if i is None:
            rows += [lens[b], 0, 0]
            continue
        if i not in offsets:
            offsets[i] = nf
            clips.append(source.clips[i])
            nf += source.lengths[i]
        rows += [lens[b], offsets[i], source.lengths[i]]
    if not clips:
        clips = [np.zeros(1, np.float32)]
    if B == 0 or N == 0:
        return out
    d, o_rows, o_clip = _upload(dev, rows, clips)
    _native.call("wekws_reverb", pcm, code, B, N, pcm.stride(0), d.data_ptr() + o_rows, d.data_ptr() + o_clip, out,
                 out.stride(0), device=dev)
    return out


def launch_noise(pcm: torch.Tensor, lens: Sequence[int], picks, source: AugmentSource,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """The device half of ``add_noise``: picks[b] = (index, start or None, snr) or None.  ``out`` None = a new float32
    (B, N) tensor; ``out`` may be ``pcm`` itself when pcm is float32."""
    pcm, code, _ = _native.pcm_rows(pcm, "add_noise", one_d=False)
    B, N = pcm.shape
    dev = pcm.device
    if out is None:
        out = torch.empty(B, N, dtype=torch.float32, device=dev)
    whole, clips, rows, snr, nf = {}, [], [], [], 0
    for b, p in enumerate(picks):
        n = lens[b]
        if p is None or n == 0:                  # an empty row: the draws were made, nothing is added
            rows += [n, 0, 0]
            snr.append(0.0)
            continue
        i, start, s = p
        if start is not None:                    # a segment of a longer clip
            rows += [n, nf, n]
            clips.append(source.clips[i][start:start + n])
            nf += n
        else:                                    # the whole clip, repeated up to n samples
            if i not in whole:
                whole[i] = nf
                clips.append(source.clips[i])
                nf += source.lengths[i]
            rows += [n, whole[i], source.lengths[i]]
        snr.append(float(s))
    if B == 0 or N == 0:
        return out
    if not clips:
        clips = [np.zeros(1, np.float32)]
    d, o_rows, o_clip = _upload(dev, rows, clips, snr)
    _native.call("wekws_add_noise", pcm, code, B, N, pcm.stride(0), d.data_ptr() + o_rows, d, d.data_ptr() + o_clip,
                 out, out.stride(0), device=dev)
    return out


def reverb(pcm: torch.Tensor, lengths, source: AugmentSource, prob: float, rng=random) -> torch.Tensor:
    """processor.add_reverb on a batch: pcm (B, N) int16 or float32 CUDA tensor at int16 scale, row b = its first
    lengths[b] samples.  Each row in turn makes add_reverb's draws from ``rng``; a selected row is convolved with its
    RIR, normalised to unit energy, and truncated to its length.  Returns a new float32 (B, N) tensor: unselected rows
    and samples past a row's length are the input, converted exactly."""
    pcm, lens = _check(pcm, lengths, "reverb")
    picks = [draw_reverb(n, source, prob, rng, b) for b, n in enumerate(lens)]
    return launch_reverb(pcm, lens, picks, source)


def add_noise(pcm: torch.Tensor, lengths, source: AugmentSource, prob: float, rng=random) -> torch.Tensor:
    """processor.add_noise on a batch: pcm as ``reverb`` takes it.  Each row in turn makes add_noise's draws from
    ``rng``; a selected row gets its noise segment at the drawn SNR.  Returns a new float32 (B, N) tensor: unselected
    rows, empty rows and samples past a row's length are the input, converted exactly."""
    pcm, lens = _check(pcm, lengths, "add_noise")
    picks = [draw_noise(n, source, prob, rng) for n in lens]
    return launch_noise(pcm, lens, picks, source)
