"""Training-audio augmentation on the device (csrc/augment.cu): reverb against its float64 evaluation and the
reference's outputs, additive noise against the float64 formula and the reference, and TrainFeatures with sources
against the hey_snips chain written from the reference (oracle/make_augment_golden.py)."""
import json
import random

import numpy as np
import pytest
import torch

from oracle import kws_augment_oracle as A
from tests.conftest import golden
from tests.test_augment_host import (CHAINS, TOL_FBANK_MAX, TOL_FBANK_MEAN, chain_f64, golden_rows, noise_rows,
                                     reverb_rows_f64, sources, stage_picks)
from wekws_b200 import AugmentSource, TrainFeatures, _native, add_noise, reverb

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pcm(dtype):
    pcm, lens = A.audio()
    x = torch.from_numpy(pcm)
    return (x if dtype == "int16" else x.float()), lens


def _launches(fn):
    n0 = _native.launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, _native.launch_count() - n0


def _ulp_check(got, want, what):
    """|got - want| within 1 ulp of want's float32 rounding (plus 1e-12 of the row's scale for exact cancellation)."""
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got.astype(np.float64) - want)
    bad = err > ulp + 1e-12 * np.abs(want).max()
    assert not bad.any(), (what, int(bad.sum()), float(err.max()))
    return err


@pytest.mark.parametrize("dtype", ["int16", "float32"])
def test_reverb_golden_rows(dtype):
    g = golden("augment")
    pcm, lens = _pcm(dtype)
    rv, _ = sources()
    y, n = _launches(lambda: reverb(pcm.to(DEV), lens, rv, float(g["rv_prob"]), rng=random.Random(int(g["rv_seed"]))))
    assert n == 1 and y.dtype == torch.float32 and y.shape == pcm.shape
    y = y.cpu().numpy()
    picks = stage_picks(g, "reverb")
    truth, ref = reverb_rows_f64(picks), golden_rows(g, "rv_out", picks, lens)
    x = pcm.float().numpy()
    for b, p in enumerate(picks):
        if p is None:
            assert np.array_equal(y[b].view(np.uint32), x[b].view(np.uint32)), b          # bit for bit
            continue
        n = lens[b]
        err = _ulp_check(y[b, :n], truth[b], b)
        assert err.max() <= np.abs(ref[b] - truth[b]).max(), b      # never further than the reference's float32 FFT
        assert np.array_equal(y[b, n:], x[b, n:])                   # past the row: the input


@pytest.mark.parametrize("dtype", ["int16", "float32"])
def test_reverb_ragged_tiles_and_long_rirs(dtype):
    """Rows across several 2048-output tiles and 512-tap chunks, RIRs shorter and longer than the rows, on a strided
    view."""
    g = torch.Generator().manual_seed(3)
    lens = [20000, 1, 2047, 2048, 2049, 9000, 16001, 513]
    N = 20480
    base = (torch.randn(len(lens), N + 64, generator=g) * 3000).round().clamp(-32768, 32767)
    base = base.to(torch.int16) if dtype == "int16" else base
    pcm = base[:, 32:32 + N]
    rng = np.random.default_rng(4)
    rirs = [("r16000", A.wav_bytes((rng.standard_normal(16000) * np.exp(-np.arange(16000) / 3000)).astype(np.float32))),
            ("r700", A.wav_bytes(np.round(rng.standard_normal(700) * 5000).astype(np.int16))),
            ("r1", A.wav_bytes(np.array([-3.5], np.float32)))]
    src = AugmentSource(rirs, rir=True)
    r = random.Random(11)
    y = reverb(pcm.to(DEV), lens, src, 1.0, rng=r).cpu().numpy()
    r = random.Random(11)
    picks = [r.randint(0, 2) if r.random() < 1.0 else None for _ in lens]
    assert set(picks) == {0, 1, 2}
    x = pcm.float().numpy()
    for b, n in enumerate(lens):
        _ulp_check(y[b, :n], A.reverb_f64(x[b, :n], src.clips[picks[b]]), b)
        assert np.array_equal(y[b, n:], x[b, n:])


@pytest.mark.parametrize("dtype", ["int16", "float32"])
def test_noise_golden_rows(dtype):
    g = golden("augment")
    pcm, lens = _pcm(dtype)
    _, nz = sources()
    y, n = _launches(lambda: add_noise(pcm.to(DEV), lens, nz, float(g["nz_prob"]),
                                       rng=random.Random(int(g["nz_seed"]))))
    assert n == 1
    y = y.cpu().numpy()
    picks = stage_picks(g, "noise")
    f64, ref = noise_rows(picks), golden_rows(g, "nz_out", picks, lens)
    x = pcm.float().numpy()
    for b, p in enumerate(picks):
        if p is None:
            assert np.array_equal(y[b].view(np.uint32), x[b].view(np.uint32)), b
            continue
        n = lens[b]
        got = y[b, :n].astype(np.float64)
        scale = np.abs(x[b, :n]) + np.abs(f64[b] - x[b, :n])              # |x| + |gain s|
        assert (np.abs(got - f64[b]) <= 3 * np.spacing(scale.astype(np.float32))).all(), b
        rms = np.sqrt(np.mean(f64[b] ** 2))
        assert np.abs(got - ref[b]).max() <= 1e-5 * rms, b
        assert np.array_equal(y[b, n:], x[b, n:])


def test_noise_empty_row_and_reverb_refusal():
    _, nz = sources()
    rv, _ = sources()
    pcm = torch.ones(2, 100, dtype=torch.int16, device=DEV)
    y = add_noise(pcm, [0, 100], nz, 1.0, rng=random.Random(2))
    assert torch.equal(y[0], pcm[0].float()) and not torch.equal(y[1], pcm[1].float())
    with pytest.raises(ValueError, match="row 0"):
        reverb(pcm, [0, 100], rv, 1.0, rng=random.Random(2))
    with pytest.raises(RuntimeError, match="CUDA"):
        reverb(pcm.cpu(), [0, 100], rv, 1.0)


@pytest.mark.parametrize("name", CHAINS)
@pytest.mark.parametrize("dtype", ["int16", "float32"])
def test_train_features_with_sources_match_reference_chain(name, dtype):
    g = golden("augment")
    conf = json.loads(str(g[name + "_conf"]))
    rv, nz = sources()
    tf = TrainFeatures.from_config(conf, reverb_source=rv, noise_source=nz)
    pcm, lens = _pcm(dtype)
    batch = tf(pcm.to(DEV), lens, 16000, json.loads(str(g[name + "_labels"])), g[name + "_keys"].tolist(),
               rng=A.Recorder(int(g[name + "_rng_seed"])), generator=torch.Generator().manual_seed(int(g["gen_seed"])))
    assert batch["keys"] == g[name + "_out_keys"].tolist()
    assert np.array_equal(batch["feats_lengths"].numpy(), g[name + "_feats_lengths"])
    assert np.array_equal(batch["target"].numpy(), g[name + "_target"])
    got, want = batch["feats"].cpu().numpy(), g[name + "_feats"]
    assert got.shape == want.shape and np.array_equal(got == 0, want == 0)       # masks and padding exact
    err = np.abs(got - want)
    print(f"{name} {dtype}: max {err.max():.2e} mean {err.mean():.2e}")
    if err.max() <= TOL_FBANK_MAX and err.mean() <= TOL_FBANK_MEAN:
        return
    truth = chain_f64(g, name, tf)
    e_ref, e_out = np.abs(want - truth), np.abs(got - truth)
    assert e_out.max() <= max(TOL_FBANK_MAX, 1.5 * e_ref.max()), (e_out.max(), e_ref.max())
    assert e_out.mean() <= max(TOL_FBANK_MEAN, 1.5 * e_ref.mean()), (e_out.mean(), e_ref.mean())


def test_train_features_without_sources_unchanged():
    """No sources, or sources at probability 0, or the cv split: the same draws and bit-identical features."""
    g = golden("augment")
    conf = dict(json.loads(str(g["snips_sa_conf"])))
    rv, nz = sources()
    pcm, lens = _pcm("int16")
    args = (pcm.to(DEV), lens, 16000, [0] * len(lens), [str(i) for i in range(len(lens))])
    outs, states = [], []
    for tf in (TrainFeatures.from_config(conf),
               TrainFeatures.from_config(dict(conf, reverb_prob=0, noise_prob=0), reverb_source=rv, noise_source=nz)):
        r = random.Random(5)
        outs.append(tf(*args, rng=r, generator=torch.Generator().manual_seed(1))["feats"])
        states.append(r.getstate())
    assert torch.equal(outs[0], outs[1]) and states[0] == states[1]
    cv = [TrainFeatures.from_config(conf, "cv", *s)(*args, generator=torch.Generator().manual_seed(1))["feats"]
          for s in ((None, None), (rv, nz))]
    assert torch.equal(cv[0], cv[1])
    # and with sources the features differ
    tf = TrainFeatures.from_config(dict(conf, reverb_prob=1.0, noise_prob=1.0), reverb_source=rv, noise_source=nz)
    aug = tf(*args, rng=random.Random(5), generator=torch.Generator().manual_seed(1))["feats"]
    assert not torch.equal(aug, outs[0])
