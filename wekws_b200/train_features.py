"""Training batches on the device: the data side of stage 2 of the recipes.

In the reference, data-loader workers build each training batch one utterance at a time on the CPU
(wekws/dataset/dataset.py Dataset(), and wekws/dataset/init_dataset.py on top of wenet's equivalent):

    resample -> [add_reverb -> add_noise] -> compute_fbank / compute_mfcc (dither) -> spec_aug -> context_expansion
    -> frame_skip -> padding

``TrainFeatures`` runs that chain on a batch of decoded PCM: the resampler (csrc/resample.cu), reverberation and
additive noise when it is given their sources (csrc/augment.cu, wekws_b200/augment.py), the dithered Fbank /
MFCC kernel (csrc/fbank.cu, noise from csrc/dither.cuh), SpecAugment (csrc/spec_aug.cu) and context expansion / frame
skip (csrc/stream_frontend.cu), then ``padding``'s ordering.  It returns the batch dict ``Executor.train`` reads, with
the features already on the device.  Deliberate differences from the reference:
  * the dither noise is not torch.randn's (no device generator can reproduce it) but a documented function of a seed
    drawn from torch's generator (include/wekws_b200.h), so torch.manual_seed still makes a run reproducible;
  * ``speed_perturb: true`` is refused: the reference's sox effects are gone from the torchaudio it pins, and no
    shipped config enables it.
"""
from __future__ import annotations

import random
from typing import List, Optional, Sequence

import torch

from . import _native
from .augment import AugmentSource, draw_noise, draw_reverb, launch_noise, launch_reverb
from .frontend import Fbank, Mfcc, Resample
from .postproc import context_expansion

FBANK_RATE = 16000


def draw_spec_aug_masks(frames: Sequence[int], dim: int, num_t_mask: int = 2, num_f_mask: int = 2, max_t: int = 50,
                        max_f: int = 10, rng=random) -> List[List[int]]:
    """The masks processor.spec_aug draws for each row in turn, with the same ``rng`` calls in the same order:
    num_t_mask x (randint(0, frames_b - 1), randint(1, max_t)), then num_f_mask x (randint(0, dim - 1),
    randint(1, max_f)).  Row b -> [t_start, t_end, ..., f_start, f_end, ...] with end = min(limit, start + length).
    A row with no frames raises ValueError, as the reference's randint(0, -1) does."""
    return [draw_spec_aug_row(n, dim, num_t_mask, num_f_mask, max_t, max_f, rng, b) for b, n in enumerate(frames)]


def draw_spec_aug_row(n: int, dim: int, num_t_mask: int = 2, num_f_mask: int = 2, max_t: int = 50, max_f: int = 10,
                      rng=random, row: int = 0) -> List[int]:
    """The masks processor.spec_aug draws for one utterance of n frames (row ``row`` of its batch, for the error
    message): one row of draw_spec_aug_masks."""
    n = int(n)
    if n <= 0:
        raise ValueError(f"spec_aug: row {row} has no frames")
    out = []
    for _ in range(num_t_mask):
        start = rng.randint(0, n - 1)
        length = rng.randint(1, max_t)
        out += [start, min(n, start + length)]
    for _ in range(num_f_mask):
        start = rng.randint(0, dim - 1)
        length = rng.randint(1, max_f)
        out += [start, min(dim, start + length)]
    return out


def spec_aug(feats: torch.Tensor, frames: Sequence[int], num_t_mask: int = 2, num_f_mask: int = 2, max_t: int = 50,
             max_f: int = 10, rng=random) -> torch.Tensor:
    """processor.spec_aug on a batch, in place: feats (B, T, D) float32 CUDA, row b's first frames[b] (host ints)
    frames are its utterance.  The masks come from ``rng`` (Python's ``random`` by default) in the reference's order,
    so with the same random state they are the reference's; one small asynchronous copy sends them up and one launch
    writes the zeros.  Returns feats."""
    if not feats.is_cuda:
        raise RuntimeError("wekws_b200.spec_aug runs on CUDA (sm_90a) only; got a CPU tensor (no CPU fallback)")
    if feats.dim() != 3 or feats.dtype != torch.float32 or not feats.is_contiguous():
        raise ValueError("feats must be a contiguous (B, T, D) float32 tensor")
    B, T, D = feats.shape
    frames = [int(n) for n in frames]
    if len(frames) != B or any(n > T for n in frames):
        raise ValueError(f"frames must be {B} values of at most {T}")
    masks = draw_spec_aug_masks(frames, D, num_t_mask, num_f_mask, max_t, max_f, rng)
    return _apply_spec_aug(feats, frames, masks, num_t_mask, num_f_mask)


def _apply_spec_aug(feats: torch.Tensor, frames: List[int], masks: List[List[int]], num_t_mask: int,
                    num_f_mask: int) -> torch.Tensor:
    B, T, D = feats.shape
    if B == 0 or num_t_mask + num_f_mask == 0:
        return feats
    table = torch.tensor(frames + [v for row in masks for v in row], dtype=torch.int32).pin_memory()
    dev = feats.device
    with torch.cuda.device(dev):
        d_table = table.to(dev, non_blocking=True)
    _native.call("wekws_spec_aug", feats, d_table, B, T, D, d_table.data_ptr() + 4 * B, int(num_t_mask),
                 int(num_f_mask), device=dev)
    return feats


class TrainFeatures:
    """The reference's training data chain after decoding, for one batch of PCM at a time.

    ``feat_type`` 'fbank' or 'mfcc'; ``feat_conf`` the keys compute_fbank / compute_mfcc take (num_mel_bins,
    num_ceps, frame_length, frame_shift, dither; their defaults when absent).  ``spec_aug_conf`` None = no SpecAugment.
    ``context`` (left, right) or None; ``frame_skip`` >= 1.  ``reverb_source`` / ``noise_source``: AugmentSource
    banks (Dataset()'s reverb_lmdb / noise_lmdb), applied after resampling with ``reverb_prob`` / ``noise_prob``; a
    stage runs only when its source is given and its probability is above 0, as Dataset() adds it."""

    def __init__(self, feat_type: str = "fbank", feat_conf: Optional[dict] = None, resample_rate: int = FBANK_RATE,
                 spec_aug_conf: Optional[dict] = None, context=None, frame_skip: int = 1,
                 reverb_source: Optional[AugmentSource] = None, reverb_prob: float = 0.0,
                 noise_source: Optional[AugmentSource] = None, noise_prob: float = 0.0):
        conf = dict(feat_conf or {})
        kw = dict(frame_length=float(conf.get("frame_length", 25)), frame_shift=float(conf.get("frame_shift", 10)))
        if feat_type == "fbank":
            self.frontend = Fbank(int(conf.get("num_mel_bins", 23)), **kw)
        elif feat_type == "mfcc":
            self.frontend = Mfcc(int(conf.get("num_ceps", 80)), int(conf.get("num_mel_bins", 80)), **kw)
        else:
            raise ValueError(f"feature type {feat_type!r}: the recipes use 'fbank' or 'mfcc'")
        if int(resample_rate) != FBANK_RATE:
            raise NotImplementedError(f"resample_rate {resample_rate}: the Fbank kernel runs at {FBANK_RATE} Hz only")
        self.feat_type = feat_type
        self.dither = float(conf.get("dither", 0.0))
        self.resample_rate = int(resample_rate)
        self.spec_aug_conf = None if spec_aug_conf is None else dict(spec_aug_conf)
        self.context = None if context is None else (int(context[0]), int(context[1]))
        self.frame_skip = int(frame_skip)
        if self.frame_skip < 1:
            raise ValueError(f"frame_skip must be >= 1, got {frame_skip}")
        self.reverb_source = reverb_source if reverb_source is not None and float(reverb_prob) > 0 else None
        self.reverb_prob = float(reverb_prob)
        self.noise_source = noise_source if noise_source is not None and float(noise_prob) > 0 else None
        self.noise_prob = float(noise_prob)
        self._resamplers = {}

    @classmethod
    def from_config(cls, dataset_conf: dict, split: str = "train", reverb_source: Optional[AugmentSource] = None,
                    noise_source: Optional[AugmentSource] = None) -> "TrainFeatures":
        """Reads ``dataset_conf`` as the reference's chains do: the live schema (feats_type + fbank_conf / mfcc_conf,
        init_dataset.py) or the legacy one (feature_extraction_conf with feature_type, dataset.py Dataset());
        resample_conf (16 kHz when absent, processor.resample's default); spec_aug (on when the key is absent, as in
        Dataset()) with spec_aug_conf; context_expansion with context_expansion_conf; frame_skip.  split != 'train'
        applies init_dataset.py's evaluation overrides: no spec_aug and no speed_perturb.  Dither stays on there, as
        it does in the reference, whose overrides leave the feature config alone.  ``reverb_source`` /
        ``noise_source`` take effect with reverb_prob / noise_prob (0 when absent) in the 'train' split only: the
        held-out sets of the recipes are built without the LMDB sources."""
        conf = dict(dataset_conf)
        if split != "train":
            conf["speed_perturb"] = False
            conf["spec_aug"] = False
            reverb_source = noise_source = None
        if conf.get("speed_perturb", False):
            raise NotImplementedError("speed_perturb: the reference's sox speed effect is not available in the "
                                      "torchaudio it pins, and no shipped config enables it")
        if "feats_type" in conf:
            feat_type = conf["feats_type"]
            feat_conf = conf.get(f"{feat_type}_conf", {})
        else:
            feat_conf = dict(conf.get("feature_extraction_conf", {}))
            feat_type = feat_conf.pop("feature_type", None)
            if feat_type is None:
                raise KeyError("dataset_conf has neither feats_type nor feature_extraction_conf.feature_type")
        resample_rate = conf.get("resample_conf", {}).get("resample_rate", FBANK_RATE)
        sa = conf.get("spec_aug_conf", {}) if conf.get("spec_aug", True) else None
        context = None
        if conf.get("context_expansion", False):
            cc = conf.get("context_expansion_conf", {})
            context = (cc.get("left", 1), cc.get("right", 1))
        return cls(feat_type, feat_conf, resample_rate, sa, context, conf.get("frame_skip", 1),
                   reverb_source, conf.get("reverb_prob", 0.0), noise_source, conf.get("noise_prob", 0.0))

    def draw(self, lengths: Sequence[int], rng=random) -> dict:
        """The host draws of a batch whose rows have ``lengths`` samples at resample_rate, made utterance by utterance
        as the reference's lazy processors make them: row b's add_reverb draws, then its add_noise draws, then its
        SpecAugment masks, before row b + 1 draws anything.  Returns {'reverb': B clip indices or None, 'noise': B
        (index, start or None, snr) or None, 'masks': B mask rows (empty lists without SpecAugment)}."""
        fe, sa = self.frontend, self.spec_aug_conf
        out = {"reverb": [], "noise": [], "masks": []}
        for b, n in enumerate(int(v) for v in lengths):
            out["reverb"].append(None if self.reverb_source is None
                                 else draw_reverb(n, self.reverb_source, self.reverb_prob, rng, b))
            out["noise"].append(None if self.noise_source is None
                                else draw_noise(n, self.noise_source, self.noise_prob, rng))
            out["masks"].append([] if sa is None
                                else draw_spec_aug_row(fe.num_frames(n), fe.feature_dim, rng=rng, row=b, **sa))
        return out

    def _resampler(self, orig: int) -> Resample:
        rs = self._resamplers.get(orig)
        if rs is None:
            rs = self._resamplers[orig] = Resample(orig, self.resample_rate)
        return rs

    def __call__(self, pcm: torch.Tensor, lengths: Sequence[int], sample_rate: int, labels, keys,
                 rng=random, generator: Optional[torch.Generator] = None) -> dict:
        """pcm (B, N) int16 or float32 CUDA tensor at int16 scale (the reference's waveform * (1 << 15)), row b = its
        first lengths[b] samples (host ints), all at ``sample_rate``; labels: B ints or B token lists; keys: B
        strings.  Returns {keys, feats, target, feats_lengths, target_lengths} in padding()'s order (longest first):
        feats (B, T, D) float32 on pcm's device, the rest host tensors as padding() makes them.  ``rng`` makes the
        augmentation draws and the SpecAugment masks (see ``draw``), ``generator`` the dither seed."""
        pcm, _, _ = _native.pcm_rows(pcm, "TrainFeatures", one_d=False)
        B, N = pcm.shape
        lens = _native.host_lengths(lengths, B, N)
        if len(labels) != B or len(keys) != B:
            raise ValueError(f"labels and keys must have {B} entries")
        dev = pcm.device
        wave = pcm
        if int(sample_rate) != self.resample_rate:
            rs = self._resampler(int(sample_rate))
            wave = rs(pcm, torch.tensor(lens, dtype=torch.int32).to(dev))
            lens = [rs.output_length(n) for n in lens]
        fe = self.frontend
        frames = [fe.num_frames(n) for n in lens]
        wave = wave[:, :max(lens, default=0)]
        draws = None
        if self.reverb_source is not None or self.noise_source is not None:
            draws = self.draw(lens, rng)
            owned = int(sample_rate) != self.resample_rate          # wave is the resampler's buffer, not the caller's
            if any(p is not None for p in draws["reverb"]):
                wave, owned = launch_reverb(wave, lens, draws["reverb"], self.reverb_source), True
            if any(p is not None for p in draws["noise"]):
                wave = launch_noise(wave, lens, draws["noise"], self.noise_source,
                                    out=wave if owned and wave.dtype == torch.float32 else None)
        feats = fe(wave, lengths=torch.tensor(lens, dtype=torch.int32).to(dev), dither=self.dither,
                   generator=generator)
        if self.spec_aug_conf is not None:
            if draws is None:
                spec_aug(feats, frames, rng=rng, **self.spec_aug_conf)
            else:
                sa = self.spec_aug_conf
                _apply_spec_aug(feats, frames, draws["masks"], sa.get("num_t_mask", 2), sa.get("num_f_mask", 2))
        feat_lens = torch.tensor(frames, dtype=torch.int32)
        if self.context is not None or self.frame_skip > 1:
            left, right = self.context or (0, 0)
            feats, feat_lens = context_expansion(feats, left, right, self.frame_skip, feat_lens)
        order, batch = padding_order(feat_lens, labels, keys)
        T = int(batch["feats_lengths"][0]) if B else 0
        batch["feats"] = feats.index_select(0, order.to(dev))[:, :T].contiguous()
        return batch


def padding_order(feat_lens: torch.Tensor, labels, keys):
    """The host half of processor.padding(): order = torch.argsort(feat_lens, descending=True) (the same sort as the
    reference, ties included), and the batch dict without feats: keys and labels in that order, int labels as a (B,)
    int32 tensor with lengths 1, token lists padded with -1.  Returns (order, dict)."""
    order = torch.argsort(feat_lens, descending=True)
    idx = order.tolist()
    if idx and isinstance(labels[0], int):
        target = torch.tensor([labels[i] for i in idx], dtype=torch.int32)
        target_lens = torch.ones(len(idx), dtype=torch.int32)
    else:
        seqs = [torch.tensor(labels[i], dtype=torch.int32) for i in idx]
        target_lens = torch.tensor([len(s) for s in seqs], dtype=torch.int32)
        target = (torch.nn.utils.rnn.pad_sequence(seqs, batch_first=True, padding_value=-1) if seqs
                  else torch.zeros(0, 0, dtype=torch.int32))
    return order, {"keys": [keys[i] for i in idx], "feats": None, "target": target,
                   "feats_lengths": feat_lens[order], "target_lengths": target_lens}
