"""The training front-end on the device: the dither generator (csrc/dither.cuh) against its float64 restatement and as
a Gaussian source, the dithered Fbank / MFCC kernel against the oracle fed the same noise, SpecAugment (csrc/spec_aug.cu)
and TrainFeatures against the golden written from the reference's own chain (oracle/make_train_features_golden.py)."""
import ctypes as C
import json
import random

import numpy as np
import pytest
import torch

from oracle import kws_train_oracle as T
from tests.conftest import golden
from tests.feature_gates import check_feats
from tests.test_train_features_host import chain_f64
from wekws_b200 import Fbank, Mfcc, TrainFeatures, spec_aug, _native
from wekws_b200.frontend import draw_seed

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL_FBANK_MAX, TOL_FBANK_MEAN = 1e-3, 1e-5      # tests/test_gpu_parity.py feature tolerances
TOL_MFCC_MAX, TOL_MFCC_MEAN = 6e-3, 6e-4
CHAINS = ["ds_tcn", "mdtc", "fsmn_ctc"]


def device_noise(seed, B, frames):
    out = torch.empty(B, frames, 400, device=DEV)
    _native.check(_native.lib().wekws_dither_noise(seed, B, frames, C.c_void_p(out.data_ptr()),
                                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)),
                  "wekws_dither_noise")
    return out


def test_noise_matches_float64_restatement():
    for seed in (0, 1, 0xDEADBEEFCAFEF00D):
        dev = device_noise(seed, 5, 300).cpu().double().numpy()
        ref = T.dither_noise(seed, 5, 300)
        err = np.abs(dev - ref).max()
        print(f"seed {seed:#x}: max |device - float64| = {err:.3e}")
        assert err <= 1e-6


def test_noise_statistics():
    n = device_noise(12345, 64, 656)                     # 64 * 656 * 400 = 16.8 M >= 2^24 normals
    assert n.numel() >= 1 << 24
    x = n.double()
    mean, var = float(x.mean()), float(x.var())
    assert abs(mean) < 1e-3 and abs(var - 1) < 2e-3, (mean, var)

    def corr(a, b):
        a, b = a.reshape(-1) - a.mean(), b.reshape(-1) - b.mean()
        return float((a * b).mean() / (a.std() * b.std()))
    assert abs(corr(x[..., :-1], x[..., 1:])) < 2e-3                     # neighbouring samples
    assert abs(corr(x[:, :-1, 160:], x[:, 1:, :240])) < 2e-3             # the same signal sample in overlapping frames
    assert abs(corr(x[:-1], x[1:])) < 2e-3                               # neighbouring rows
    from scipy import stats
    p = stats.kstest(n.reshape(-1)[: 1 << 24].cpu().numpy().astype(np.float64), "norm").pvalue
    assert p > 1e-3, p
    other = device_noise(12346, 64, 656)
    assert (other != n).float().mean() > 0.99


def _batch(dtype, B=5, N=16000 + 777):
    g = torch.Generator().manual_seed(8)
    pcm = (torch.randn(B, N, generator=g) * 2500).clamp(-32768, 32767)
    pcm = pcm.round().to(torch.int16) if dtype == "int16" else pcm
    lens = [N, 400, N - 1000, 10000, N - 161]
    return pcm, lens[:B]


@pytest.mark.parametrize("dtype", ["int16", "float32"])
@pytest.mark.parametrize("kind", ["fbank40", "fbank80", "mfcc80", "mfcc40x13", "fbank23", "fbank128", "mfcc128x128"])
def test_dithered_features_match_oracle_with_dumped_noise(dtype, kind):
    pcm, lens = _batch(dtype)
    mfccs = {"mfcc80": (80, 80), "mfcc40x13": (13, 40), "mfcc128x128": (128, 128)}
    fe = Fbank(int(kind[5:])) if kind.startswith("fbank") else Mfcc(*mfccs[kind])
    seed = draw_seed(torch.Generator().manual_seed(5))
    out = fe(pcm.to(DEV), lengths=torch.tensor(lens, dtype=torch.int32), dither=1.0,
             generator=torch.Generator().manual_seed(5)).cpu()
    undithered = fe(pcm.to(DEV), lengths=torch.tensor(lens, dtype=torch.int32)).cpu()
    m = out.shape[1]
    noise = device_noise(seed, len(lens), m).cpu()
    tmax, tmean = (TOL_FBANK_MAX, TOL_FBANK_MEAN) if kind.startswith("fbank") else (TOL_MFCC_MAX, TOL_MFCC_MEAN)
    for b, n in enumerate(lens):
        k = fe.num_frames(n)
        x = pcm[b, :n].float()
        ref = (T.fbank(x, fe.num_mel_bins, noise[b]) if kind.startswith("fbank")
               else T.mfcc(x, fe.num_ceps, fe.num_mel_bins, noise[b]))
        err = (out[b, :k] - ref).abs()
        assert float(err.max()) <= tmax and float(err.mean()) <= tmean, (b, float(err.max()), float(err.mean()))
        assert torch.count_nonzero(out[b, k:]) == 0
    assert not torch.equal(out, undithered)                               # the noise is really added


@pytest.mark.parametrize("mfcc", [False, True])
def test_seeded_repeatability_and_dither_zero_path(mfcc):
    pcm, lens = _batch("int16")
    fe = Mfcc(80, 80) if mfcc else Fbank(40)
    x, L = pcm.to(DEV), torch.tensor(lens, dtype=torch.int32)
    a = fe(x, lengths=L, dither=1.0, generator=torch.Generator().manual_seed(9))
    b = fe(x, lengths=L, dither=1.0, generator=torch.Generator().manual_seed(9))
    c = fe(x, lengths=L, dither=1.0, generator=torch.Generator().manual_seed(10))
    assert torch.equal(a, b) and not torch.equal(a, c)
    torch.manual_seed(3)
    d = fe(x, lengths=L, dither=1.0)
    torch.manual_seed(3)
    assert torch.equal(d, fe(x, lengths=L, dither=1.0))                   # torch.manual_seed governs the default
    plain = fe(x, lengths=L)
    n0 = _native.launch_count()
    zero = fe(x, lengths=L, dither=0.0, generator=torch.Generator().manual_seed(9))
    torch.cuda.synchronize()
    assert _native.launch_count() - n0 == 1
    assert torch.equal(zero, plain)


def test_spec_aug_matches_golden_exactly():
    g = golden("train_features")
    x_in, frames = T.spec_aug_input()
    zero = np.unpackbits(g["sa_zero"], count=x_in.size).reshape(x_in.shape).astype(bool)
    want = np.where(zero, np.float32(0), x_in)              # the reference's result: zeros, the input elsewhere
    x = torch.from_numpy(x_in).to(DEV)
    n0 = _native.launch_count()
    y = spec_aug(x, frames, rng=random.Random(int(g["sa_rng_seed"])))
    torch.cuda.synchronize()
    assert _native.launch_count() - n0 == 1 and y is x
    got = y.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))       # exact zeros, the rest bitwise untouched
    with pytest.raises(ValueError, match="row 2"):
        spec_aug(torch.zeros(3, 10, 4, device=DEV), [4, 10, 0])


@pytest.mark.parametrize("name", CHAINS)
@pytest.mark.parametrize("dtype", ["int16", "float32"])
def test_train_features_match_reference_chain(name, dtype):
    g = golden("train_features")
    conf = json.loads(str(g[name + "_conf"]))
    tf = TrainFeatures.from_config(conf)
    pcm_np, lens = T.golden_audio()
    pcm = torch.from_numpy(pcm_np)
    pcm = pcm if dtype == "int16" else pcm.float()
    labels = json.loads(str(g[name + "_labels"]))
    batch = tf(pcm.to(DEV), lens, 16000, labels, g[name + "_keys"].tolist(),
               rng=random.Random(int(g["rng_seed"])), generator=torch.Generator().manual_seed(int(g["gen_seed"])))
    assert batch["keys"] == g[name + "_out_keys"].tolist()
    assert np.array_equal(batch["feats_lengths"].numpy(), g[name + "_feats_lengths"])
    assert np.array_equal(batch["target"].numpy(), g[name + "_target"])
    assert np.array_equal(batch["target_lengths"].numpy(), g[name + "_target_lengths"])
    feats, want = batch["feats"], g[name + "_feats"]
    assert feats.is_cuda and tuple(feats.shape) == want.shape
    got = feats.cpu().numpy()
    assert np.array_equal(got == 0, want == 0)                          # masks and padding exact
    is_mfcc = name == "mdtc"
    tmax, tmean = (TOL_MFCC_MAX, TOL_MFCC_MEAN) if is_mfcc else (TOL_FBANK_MAX, TOL_FBANK_MEAN)
    err = np.abs(got - want)
    if err.max() <= tmax and err.mean() <= tmean:
        return
    # tonal audio: the reference's own float32 rounding exceeds the tolerance (tests/test_gpu_parity.py _check_feats);
    # then the kernel must be at least as close to the chain's float64 evaluation as the reference is
    truth = chain_f64(g, name)
    e_ref, e_out = np.abs(want - truth), np.abs(got - truth)
    assert e_out.max() <= max(tmax, 1.5 * e_ref.max()), (e_out.max(), e_ref.max())
    assert e_out.mean() <= max(tmean, 1.5 * e_ref.mean()), (e_out.mean(), e_ref.mean())


def test_train_features_default_conf_is_fbank23():
    """TrainFeatures with an empty feat_conf takes compute_fbank's defaults: 23 mel bins, no dither; its features are
    the Fbank(23) kernel's, bit for bit, in padding()'s order."""
    pcm, lens = _batch("int16")
    tf = TrainFeatures(feat_conf={})
    assert tf.frontend.feature_dim == 23 and tf.dither == 0.0
    batch = tf(pcm.to(DEV), lens, 16000, [0] * len(lens), [str(i) for i in range(len(lens))])
    want = Fbank(23)(pcm.to(DEV), lengths=torch.tensor(lens, dtype=torch.int32)).cpu()
    order = [int(k) for k in batch["keys"]]
    T_max = int(batch["feats_lengths"][0])
    assert torch.equal(batch["feats"].cpu(), want[order, :T_max])
    for b, n in enumerate(lens):
        ref = T.fbank(pcm[b, :n].float(), 23)
        check_feats(want[b, :ref.shape[0]].numpy(), ref.numpy(), ("fbank23", b), pcm[b, :n].float(), num_mel_bins=23)


def test_train_features_cv_split_and_resampled_input():
    g = golden("train_features")
    conf = json.loads(str(g["ds_tcn_conf"]))
    pcm_np, lens = T.golden_audio()
    pcm = torch.from_numpy(pcm_np).to(DEV)
    args = (lens, 16000, [0] * len(lens), [str(i) for i in range(len(lens))])
    tv = TrainFeatures.from_config(conf, split="cv")
    a = tv(pcm, *args, generator=torch.Generator().manual_seed(1))
    assert torch.count_nonzero(a["feats"][0]) == a["feats"][0].numel()      # no SpecAugment zeros in cv
    # 32 kHz audio goes through the resampler before the front-end
    up = torch.repeat_interleave(pcm, 2, dim=1)
    b = tv(up, [2 * n for n in lens], 32000, *args[2:], generator=torch.Generator().manual_seed(1))
    assert b["feats_lengths"].tolist() == a["feats_lengths"].tolist()
