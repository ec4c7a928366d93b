"""Host-side pieces of the training front-end (no GPU): the dither generator's known answers, the noisy oracle against
torchaudio with torch.randn patched, SpecAugment's host mask draws against processor.spec_aug, TrainFeatures.from_config
on the recipes' dataset_conf, padding()'s order and labels, and the zero-frame refusal."""
import glob
import json
import os
import random
import sys
from unittest import mock

import numpy as np
import pytest
import torch

from oracle import kws_train_oracle as T
from tests.conftest import REFERENCE, golden, have_reference
from wekws_b200 import Fbank, Mfcc, TrainFeatures
from wekws_b200.train_features import draw_spec_aug_masks, padding_order

TOL_FBANK = 1e-3          # tests/test_oracle_pinned.py: the oracle against kaldi.fbank
TOL_MFCC = 2e-4           # tests/test_oracle_pinned.py: the oracle against kaldi.mfcc
TOL_FEAT = {"ds_tcn": (1e-3, 1e-5), "fsmn_ctc": (1e-3, 1e-5), "mdtc": (6e-3, 6e-4)}   # test_gpu_parity.py (max, mean)
CHAINS = ["ds_tcn", "mdtc", "fsmn_ctc"]


def _processor():
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    from wekws.dataset import processor
    return processor


def test_philox_known_answers():
    w = T.philox4x32_10(np.zeros(4, np.uint32), (0, 0))
    assert [f"{x:08x}" for x in w] == ["6627e8d5", "e169c58d", "bc57ac4c", "9b00dbd8"]
    ctr = np.array([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], np.uint32)
    w = T.philox4x32_10(ctr, (0xa4093822, 0x299f31d0))
    assert [f"{x:08x}" for x in w] == ["d16cfe09", "94fdcceb", "5001e420", "24126ea1"]


def test_noise_layout_is_counter_based():
    """Sample j of frame f of row b depends on (seed, b, f, j) only: a sub-batch gives the same values."""
    big = T.dither_noise(77, 3, 9)
    assert np.array_equal(T.dither_noise(77, 2, 4), big[:2, :4])
    assert not np.allclose(T.dither_noise(78, 1, 1), big[:1, :1])
    assert np.abs(big).max() < 5.9


@pytest.mark.parametrize("kind", ["fbank40", "fbank80", "mfcc80"])
def test_noisy_oracle_matches_torchaudio(kind):
    import torchaudio.compliance.kaldi as kaldi
    g = torch.Generator().manual_seed(3)
    pcm = (torch.randn(12345, generator=g) * 3000).round()
    m = T.O.num_frames(pcm.numel())
    noise = torch.from_numpy(T.dither_noise(2024, 1, m)[0]).float()
    with mock.patch.object(torch, "randn", lambda *a, **k: noise.clone()):
        if kind == "mfcc80":
            ref = kaldi.mfcc(pcm.unsqueeze(0), num_ceps=80, num_mel_bins=80, frame_length=25, frame_shift=10,
                             dither=1.0, energy_floor=0.0, sample_frequency=16000)
        else:
            ref = kaldi.fbank(pcm.unsqueeze(0), num_mel_bins=int(kind[5:]), frame_length=25, frame_shift=10,
                              dither=1.0, energy_floor=0.0, sample_frequency=16000)
    out = T.mfcc(pcm, 80, 80, noise) if kind == "mfcc80" else T.fbank(pcm, int(kind[5:]), noise)
    assert (out - ref).abs().max() <= (TOL_MFCC if kind == "mfcc80" else TOL_FBANK)
    undithered = T.mfcc(pcm, 80, 80) if kind == "mfcc80" else T.fbank(pcm, int(kind[5:]))
    assert (undithered - ref).abs().max() > 1e-3          # the noise is really there


@pytest.mark.skipif(not have_reference(), reason="reference checkout not present")
@pytest.mark.parametrize("conf", [(2, 2, 50, 10), (1, 1, 20, 40), (3, 0, 5, 1), (0, 2, 50, 30)])
def test_host_masks_equal_processor_spec_aug(conf):
    processor = _processor()
    nt, nf, mt, mf = conf
    frames, D = [120, 37, 5, 1, 64], 40
    random.seed(31)
    ref = [next(processor.spec_aug(iter([{"feat": torch.ones(n, D)}]), nt, nf, mt, mf))["feat"] for n in frames]
    masks = draw_spec_aug_masks(frames, D, nt, nf, mt, mf, rng=random.Random(31))
    for n, y, row in zip(frames, ref, masks):
        x = torch.ones(n, D)
        for i in range(nt):
            x[row[2 * i]:row[2 * i + 1], :] = 0
        for i in range(nt, nt + nf):
            x[:, row[2 * i]:row[2 * i + 1]] = 0
        assert torch.equal(x, y)


def test_zero_frame_row_is_refused():
    with pytest.raises(ValueError, match="row 1"):
        draw_spec_aug_masks([5, 0, 3], 40)


def _shipped_confs():
    confs = {f"golden:{n}": json.loads(str(golden("train_features")[n + "_conf"])) for n in CHAINS}
    if have_reference():
        import yaml
        for path in sorted(glob.glob(os.path.join(REFERENCE, "examples", "*", "s0", "conf", "*.yaml"))):
            confs[os.path.relpath(path, REFERENCE)] = yaml.safe_load(open(path))["dataset_conf"]
    return confs


@pytest.mark.parametrize("split", ["train", "cv"])
def test_from_config_on_recipe_configs(split):
    for name, conf in _shipped_confs().items():
        tf = TrainFeatures.from_config(conf, split)
        legacy = "feats_type" not in conf
        fc = conf["feature_extraction_conf"] if legacy else conf[conf["feats_type"] + "_conf"]
        ftype = fc["feature_type"] if legacy else conf["feats_type"]
        assert tf.feat_type == ftype, name
        assert isinstance(tf.frontend, Mfcc if ftype == "mfcc" else Fbank)
        assert tf.frontend.num_mel_bins == fc["num_mel_bins"]
        if ftype == "mfcc":
            assert tf.frontend.num_ceps == fc["num_ceps"]
        assert tf.dither == fc.get("dither", 0.0) == 1.0, name      # every recipe dithers, cv included
        on = split == "train" and conf.get("spec_aug", True)
        assert tf.spec_aug_conf == (conf.get("spec_aug_conf", {}) if on else None), name
        ctx = conf.get("context_expansion_conf", {}) if conf.get("context_expansion", False) else None
        assert tf.context == (None if ctx is None else (ctx.get("left", 1), ctx.get("right", 1)))
        assert tf.frame_skip == conf.get("frame_skip", 1)


def test_from_config_defaults_and_refusals():
    tf = TrainFeatures.from_config({"feature_extraction_conf": {"feature_type": "fbank", "num_mel_bins": 40}})
    assert tf.spec_aug_conf == {} and tf.dither == 0.0 and tf.context is None and tf.frame_skip == 1
    with pytest.raises(NotImplementedError, match="speed_perturb"):
        TrainFeatures.from_config({"feats_type": "fbank", "fbank_conf": {}, "speed_perturb": True})
    TrainFeatures.from_config({"feats_type": "fbank", "fbank_conf": {}, "speed_perturb": True}, split="cv")
    tf = TrainFeatures.from_config({"feats_type": "fbank", "fbank_conf": {}, "reverb_prob": 0.2, "noise_prob": 0.3})
    assert tf.frontend.num_mel_bins == 23          # compute_fbank's default
    with pytest.raises(NotImplementedError):
        TrainFeatures.from_config({"feats_type": "fbank", "fbank_conf": {}, "resample_conf": {"resample_rate": 8000}})


@pytest.mark.skipif(not have_reference(), reason="reference checkout not present")
@pytest.mark.parametrize("kind", ["int", "tokens"])
def test_padding_order_and_labels_equal_processor_padding(kind):
    processor = _processor()
    lens = [30, 52, 30, 7, 52, 52, 1, 30]
    rng = np.random.default_rng(4)
    labels = ([int(v) for v in rng.integers(-1, 3, len(lens))] if kind == "int"
              else [[int(v) for v in rng.integers(0, 99, int(rng.integers(1, 7)))] for _ in lens])
    keys = [f"u{i}" for i in range(len(lens))]
    samples = [{"key": k, "label": l, "feat": torch.zeros(n, 2)} for k, l, n in zip(keys, labels, lens)]
    k, _, target, flens, tlens = next(processor.padding(iter([samples])))
    order, batch = padding_order(torch.tensor(lens, dtype=torch.int32), labels, keys)
    assert batch["keys"] == k
    assert torch.equal(batch["target"], target) and batch["target"].dtype == target.dtype
    assert torch.equal(batch["feats_lengths"], flens) and torch.equal(batch["target_lengths"], tlens)


def test_padding_order_against_golden():
    g = golden("train_features")
    for n in CHAINS:
        labels = json.loads(str(g[n + "_labels"]))
        flens = g[n + "_feats_lengths"]
        keys = g[n + "_keys"].tolist()
        # feats lengths in input order: undo the golden's order through its keys
        pos = [g[n + "_out_keys"].tolist().index(k) for k in keys]
        _, batch = padding_order(torch.tensor(flens[pos]), labels, keys)
        assert batch["keys"] == g[n + "_out_keys"].tolist()
        assert np.array_equal(batch["target"].numpy(), g[n + "_target"])
        assert np.array_equal(batch["target_lengths"].numpy(), g[n + "_target_lengths"])


def chain_f64(g, name):
    """The golden chain ``name`` evaluated in float64 by the oracle from the golden's seeds, padded and ordered as the
    golden's features."""
    pcm, lens = T.golden_audio()
    rows = T.train_chain(pcm, lens, json.loads(str(g[name + "_conf"])), int(g[name + "_seed"]), int(g["rng_seed"]))
    keys, want = g[name + "_keys"].tolist(), g[name + "_feats"]
    out = np.zeros(want.shape)
    for i, k in enumerate(g[name + "_out_keys"].tolist()):
        r = rows[keys.index(k)].numpy()
        out[i, :r.shape[0]] = r
    return out


@pytest.mark.parametrize("name", CHAINS)
def test_float64_chain_matches_golden(name):
    """The oracle's float64 chain (the fallback yardstick of the device test) reproduces the reference's masks exactly
    and its features within the feature tolerances."""
    g = golden("train_features")
    want, truth = g[name + "_feats"], chain_f64(g, name)
    assert np.array_equal(want == 0, truth == 0)
    err = np.abs(want - truth)
    tmax, tmean = TOL_FEAT[name]
    assert err.max() <= tmax and err.mean() <= tmean, (err.max(), err.mean())
