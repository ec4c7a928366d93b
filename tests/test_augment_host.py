"""Host-side pieces of the training-audio augmentation (no GPU): the float64 oracle against the reference's outputs in
tests/golden/augment.npz, the host draws against the ``random`` calls the reference made (alone and interleaved with
SpecAugment in the hey_snips chain), source decoding and the refusals."""
import json
import sys

import numpy as np
import pytest
import torch

from oracle import kws_augment_oracle as A
from oracle import kws_train_oracle as T
from tests.conftest import REFERENCE, golden, have_reference
from wekws_b200 import AugmentSource, TrainFeatures
from wekws_b200.augment import decode_wav, draw_noise, draw_reverb, snr_range

TOL_FBANK_MAX, TOL_FBANK_MEAN = 1e-3, 1e-5      # tests/test_gpu_parity.py feature tolerances
CHAINS = ["snips", "snips_sa"]


def sources():
    return AugmentSource(A.rir_items(), rir=True), AugmentSource(A.noise_items())


def stage_picks(g, kind):
    _, lens = A.audio()
    items = A.rir_items() if kind == "reverb" else A.noise_items()
    return A.replay(str(g["rv_log" if kind == "reverb" else "nz_log"]), lens, items, kind)


def golden_rows(g, key, picks, lens):
    """The golden's stored rows (the selected ones, one after the other) at int16 scale, by row."""
    flat, out, p = g[key], {}, 0
    for b, pk in enumerate(picks):
        if pk is not None:
            out[b] = flat[p:p + lens[b]].astype(np.float64) * 32768.0
            p += lens[b]
    assert p == flat.size
    return out


def reverb_rows_f64(picks):
    pcm, lens = A.audio()
    rv, _ = sources()
    return {b: A.reverb_f64(pcm[b, :lens[b]], rv.clips[i]) for b, i in enumerate(picks) if i is not None}


def noise_rows(picks, x_rows=None, f32=False):
    pcm, lens = A.audio()
    _, nz = sources()
    out = {}
    for b, pk in enumerate(picks):
        if pk is None or lens[b] == 0:
            continue
        i, start, snr = pk
        x = pcm[b, :lens[b]] if x_rows is None else x_rows[b]
        s = A.noise_segment(nz.clips[i], lens[b], start)
        out[b] = (A.noise_f32 if f32 else A.noise_f64)(x, s, snr)
    return out


def test_reverb_oracle_reproduces_golden():
    g = golden("augment")
    _, lens = A.audio()
    picks = stage_picks(g, "reverb")
    assert None in picks and {p for p in picks if p is not None} == set(range(5))     # every RIR, some rows skipped
    want = golden_rows(g, "rv_out", picks, lens)
    for b, y in reverb_rows_f64(picks).items():
        err = np.abs(want[b] - y).max()
        assert err <= 1e-5 * np.abs(y).max() + 1e-3, (b, err)       # the reference's float32 FFT


def test_noise_oracle_reproduces_golden():
    g = golden("augment")
    _, lens = A.audio()
    picks = stage_picks(g, "noise")
    want = golden_rows(g, "nz_out", picks, lens)
    got = noise_rows(picks, f32=True)
    assert set(got) == set(want)
    for b, y in got.items():
        rms = np.sqrt(np.mean(y.astype(np.float64) ** 2))
        assert np.abs(want[b] - y).max() <= 1e-5 * rms, b


def test_stage_draws_equal_reference_random_calls():
    g = golden("augment")
    _, lens = A.audio()
    rv, nz = sources()
    rec = A.Recorder(int(g["rv_seed"]))
    for b, n in enumerate(lens):
        draw_reverb(n, rv, float(g["rv_prob"]), rec, b)
    assert rec.log == json.loads(str(g["rv_log"]))
    rec = A.Recorder(int(g["nz_seed"]))
    picks = [draw_noise(n, nz, float(g["nz_prob"]), rec) for n in lens]
    assert rec.log == json.loads(str(g["nz_log"]))
    assert picks == [tuple(p) if p else None for p in stage_picks(g, "noise")]
    # every SNR range and every clip-length relation was exercised
    sel = [(b, p) for b, p in enumerate(picks) if p is not None]
    assert {snr_range(nz.keys[p[0]]) for _, p in sel} == {(0, 15), (5, 30), (5, 15)}
    assert {np.sign(nz.lengths[p[0]] - lens[b]) for b, p in sel} == {-1, 0, 1}
    assert all(lo <= p[2] <= hi for _, p in sel for lo, hi in [snr_range(nz.keys[p[0]])])


@pytest.mark.parametrize("name", CHAINS)
def test_chain_draws_interleave_as_the_reference(name):
    g = golden("augment")
    conf = json.loads(str(g[name + "_conf"]))
    rv, nz = sources()
    tf = TrainFeatures.from_config(conf, reverb_source=rv, noise_source=nz)
    assert (tf.reverb_prob, tf.noise_prob) == (0.2, 0.3)
    _, lens = A.audio()
    rec = A.Recorder(int(g[name + "_rng_seed"]))
    draws = tf.draw(lens, rec)
    assert rec.log == json.loads(str(g[name + "_log"]))
    events = g[name + "_events"]
    assert [p is not None for p in draws["reverb"]] == events[:, 0].tolist()
    assert [p is not None for p in draws["noise"]] == events[:, 1].tolist()
    assert events[:, 0].sum() >= 2 and events[:, 1].sum() >= 2
    assert all(m == [] for m in draws["masks"]) == (name == "snips")


def chain_f64(g, name, tf=None):
    """The golden chain ``name`` in float64 by the oracle: each row's reverb and noise as the logged draws chose them,
    Fbank 40 with the restated dither noise, the drawn SpecAugment masks; padded and ordered as the golden."""
    conf = json.loads(str(g[name + "_conf"]))
    rv, nz = sources()
    tf = tf or TrainFeatures.from_config(conf, reverb_source=rv, noise_source=nz)
    pcm, lens = A.audio()
    draws = tf.draw(lens, A.Recorder(int(g[name + "_rng_seed"])))
    B = len(lens)
    dn = torch.from_numpy(T.dither_noise(int(g[name + "_seed"]), B, max(T.O.num_frames(n) for n in lens)))
    rows = []
    for b, n in enumerate(lens):
        x = pcm[b, :n].astype(np.float64)
        if draws["reverb"][b] is not None:
            x = A.reverb_f64(x, rv.clips[draws["reverb"][b]])
        if draws["noise"][b] is not None:
            i, start, snr = draws["noise"][b]
            x = A.noise_f64(x, A.noise_segment(nz.clips[i], n, start), snr)
        y = T.fbank(torch.from_numpy(x), 40, dn[b, :T.O.num_frames(n)], dtype=torch.float64).numpy()
        m = draws["masks"][b]
        if m:
            y[m[0]:m[1], :] = 0
            y[:, m[2]:m[3]] = 0
        rows.append(y)
    keys, want = g[name + "_keys"].tolist(), g[name + "_feats"]
    out = np.zeros(want.shape)
    for i, k in enumerate(g[name + "_out_keys"].tolist()):
        r = rows[keys.index(k)]
        out[i, :r.shape[0]] = r
    return out


@pytest.mark.parametrize("name", CHAINS)
def test_float64_chain_matches_golden(name):
    g = golden("augment")
    want, truth = g[name + "_feats"], chain_f64(g, name)
    assert np.array_equal(want == 0, truth == 0)
    err = np.abs(want - truth)
    assert err.max() <= TOL_FBANK_MAX and err.mean() <= TOL_FBANK_MEAN, (err.max(), err.mean())


def test_source_decoding():
    stereo = np.stack([np.arange(5, dtype=np.int16), -np.arange(5, dtype=np.int16)], axis=1)
    f32 = np.linspace(-1, 1, 7).astype(np.float32)
    src = AugmentSource([("b", A.wav_bytes(stereo)), ("a", A.wav_bytes(f32))])
    assert src.keys == ["b", "a"] and src.lengths == [5, 7]                  # key order kept, lengths on the host
    assert src.clips[0].dtype == np.float32 and np.array_equal(src.clips[0], np.arange(5, dtype=np.float32))
    assert np.array_equal(src.clips[1], f32) and np.array_equal(decode_wav(A.wav_bytes(f32)), f32)

    class Lmdbish:                                   # the reference LmdbData's surface: keys + an lmdb environment
        keys = ["a", "b"]

        class db:
            @staticmethod
            def begin(write=False):
                class Txn:
                    def __enter__(self):
                        return self

                    def __exit__(self, *a):
                        return False

                    def get(self, k):
                        return {b"a": A.wav_bytes(f32), b"b": A.wav_bytes(stereo)}[k]
                return Txn()
    src = AugmentSource(Lmdbish())
    assert src.keys == ["a", "b"] and src.lengths == [7, 5]
    assert AugmentSource({"x": A.wav_bytes(f32)}).keys == ["x"]


def test_refusals():
    with pytest.raises(ValueError, match="all zeros"):
        AugmentSource([("rir_ok", A.wav_bytes(np.ones(3, np.int16))), ("rir_z", A.wav_bytes(np.zeros(9, np.int16)))],
                      rir=True)
    AugmentSource([("silence", A.wav_bytes(np.zeros(9, np.int16)))])            # an all-zero noise clip is fine
    with pytest.raises(ValueError, match="empty"):
        AugmentSource([("n", A.wav_bytes(np.zeros(0, np.int16)))])
    with pytest.raises(ValueError):
        AugmentSource([])
    try:
        import lmdb  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match="lmdb"):
            AugmentSource.from_lmdb("/nonexistent")
    rv, nz = sources()
    with pytest.raises(ValueError, match="row 4"):
        draw_reverb(0, rv, 1.0, A.Recorder(0), 4)
    assert draw_reverb(0, rv, 0.0, A.Recorder(0), 4) is None                   # an unselected empty row is fine
    # cv never augments; without sources (or with probability 0) nothing is drawn for augmentation
    conf = {"feats_type": "fbank", "fbank_conf": {}, "reverb_prob": 0.2, "noise_prob": 0.3, "spec_aug": False}
    tv = TrainFeatures.from_config(conf, "cv", reverb_source=rv, noise_source=nz)
    assert tv.reverb_source is None and tv.noise_source is None
    tf = TrainFeatures.from_config(dict(conf, noise_prob=0), reverb_source=rv, noise_source=nz)
    assert tf.reverb_source is rv and tf.noise_source is None


@pytest.mark.skipif(not have_reference(), reason="reference checkout not present")
def test_empty_row_noise_draws_equal_reference():
    """An empty utterance: add_noise still makes its draws (a start too, the clip being longer) and returns it empty."""
    import warnings
    from unittest import mock
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    from wekws.dataset import processor
    items = A.noise_items()
    rec = A.Recorder(5)

    class Stub:
        keys = [k for k, _ in items]

        def random_one(self):
            k = self.keys[rec.randint(0, len(self.keys) - 1)]
            return k, dict(items)[k]
    with mock.patch.object(processor, "random", rec), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        y = next(processor.add_noise(iter([{"key": "u", "wav": torch.zeros(1, 0)}]), Stub(), 1.0))["wav"]
    assert y.numel() == 0
    mine = A.Recorder(5)
    _, nz = sources()
    draw_noise(0, nz, 1.0, mine)
    assert mine.log == rec.log and [c[0] for c in rec.log] == ["random", "randint", "randint", "uniform"]
