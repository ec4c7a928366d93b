"""Host-side pieces of the global CMVN statistics (no GPU): the CPU oracle against the reference's golden and the
live reference, the resampler's host table against torchaudio, its compact form, the output-length formula, and
CmvnStats.from_config / scp_segment against tools/compute_cmvn_stats.py."""
import json
import math
import os
import runpy

import numpy as np
import pytest
import torch

from oracle import kws_cmvn_oracle as CO
from tests.conftest import REFERENCE, golden, have_reference
from wekws_b200 import CmvnStats, Resample, scp_segment
from wekws_b200.frontend import sinc_resample_kernel

RATE_PAIRS = [(r, 16000) for r in CO.RATES if r != 16000] + [(16000, 8000), (8000, 44100), (16000, 48000)]
TABLE_MAX_BYTES = 96 * 1024          # resample.cu kRsTableMax: compact taps as doubles + 2 N + 1 int offsets


def _torchaudio():
    try:
        import torchaudio
        from torchaudio.functional.functional import _get_sinc_resample_kernel
        return torchaudio, _get_sinc_resample_kernel
    except Exception:
        return None, None


def golden_items(case_waves=None):
    """The golden set's utterances as the tool reads them: (int16-scale float32 waveform, rate), in scp order."""
    items = []
    for i, (key, rate, n, seg) in enumerate(CO.golden_utterances()):
        wav = CO.utterance_wave(i, n)
        if seg is not None:
            wav = wav[int(float(seg[0]) * rate):int(float(seg[1]) * rate)]
        items.append((torch.from_numpy(wav.astype(np.float32)), rate))
    return items


@pytest.mark.parametrize("case", ["fbank40", "fbank80", "mfcc80"])
def test_oracle_matches_reference_golden(case):
    g = golden("cmvn_stats")
    ft, dim = ("mfcc", 80) if case == "mfcc80" else ("fbank", int(case[5:]))
    n, m32, v32, s64 = CO.collate(golden_items(), ft, dim, 16000)
    ref = json.loads(str(g[f"{case}_json"]))
    assert n == ref["frame_num"] == int(g[f"{case}_frames"])
    # the oracle's features are within the fp32 noise of kaldi.fbank's: compare the sums relative to sum |x| (x^2)
    tol = 1e-5 * n * np.abs(g[f"{case}_sum64"]).max(axis=1, keepdims=True) / n + 1e-3
    assert (np.abs(s64.numpy() - g[f"{case}_sum64"]) <= tol * np.maximum(1.0, n / 100)).all()
    assert np.allclose(m32.numpy(), ref["mean_stat"], rtol=1e-4, atol=1e-2)
    assert np.allclose(v32.numpy(), ref["var_stat"], rtol=1e-4, atol=1e-1)


def test_oracle_resample_matches_golden():
    g = golden("cmvn_stats")
    for rate in (r for r in CO.RATES if r != 16000):
        x = torch.from_numpy(g[f"rs_in_{rate}"].astype(np.float32))
        o32 = CO.resample(x, rate, 16000).numpy()
        o64 = CO.resample(x, rate, 16000, torch.float64).numpy()
        ta = g[f"rs_ta_{rate}"]
        assert o32.shape == ta.shape == o64.shape == (math.ceil(16000 * x.numel() / rate),)
        assert np.abs(o32 - ta).max() <= 4 * np.spacing(np.abs(ta).max().astype(np.float32))
        assert np.abs(o64 - g[f"rs_f64_{rate}"]).max() <= 1e-9 * np.abs(o64).max()


def test_reference_rejects_short_utterance_golden():
    assert "400" in str(golden("cmvn_stats")["short_error"])


@pytest.mark.skipif(not have_reference() or _torchaudio()[0] is None, reason="needs the reference and torchaudio")
def test_oracle_matches_live_reference_collate():
    from oracle.make_cmvn_golden import TOOL, ScriptedAudio
    import torchaudio
    items = golden_items()[:9]
    waves = {f"/w/{i}": ((w.numpy()).astype(np.int16), r) for i, (w, r) in enumerate(items)}
    audio = ScriptedAudio(waves)
    ns = runpy.run_path(TOOL, run_name="compute_cmvn_stats")
    real_info, real_load = getattr(torchaudio, "info", None), torchaudio.load
    torchaudio.info, torchaudio.load = audio.info, audio.load
    try:
        for ft, dim in (("fbank", 40), ("mfcc", 80)):
            n_r, m_r, v_r = ns["CollateFunc"](dim, ft, 16000)([(str(i), f"/w/{i}") for i in range(len(items))])
            n_o, m_o, v_o, _ = CO.collate(items, ft, dim, 16000)
            assert n_r == n_o
            assert torch.allclose(m_o, m_r, rtol=1e-5, atol=1e-2) and torch.allclose(v_o, v_r, rtol=1e-5, atol=1e-1)
    finally:
        torchaudio.load = real_load
        if real_info is None:
            del torchaudio.info
        else:
            torchaudio.info = real_info


@pytest.mark.parametrize("orig,new", RATE_PAIRS)
def test_host_table_bit_identical_to_torchaudio(orig, new):
    ta, get_kernel = _torchaudio()
    if ta is None:
        pytest.skip("torchaudio is not importable")
    k, w = sinc_resample_kernel(orig, new)
    k_ref, w_ref = get_kernel(orig, new, math.gcd(orig, new))
    assert w == w_ref and k.dtype == k_ref.dtype == torch.float32 and torch.equal(k, k_ref)
    k_o, w_o = CO.resample_kernel(orig, new)
    assert w_o == w and torch.equal(k_o, k)
    x = torch.from_numpy(CO.scripted_wave(orig, 3001).astype(np.float32))
    assert torch.equal(CO.resample(x, orig, new), ta.transforms.Resample(orig, new)(x))


@pytest.mark.parametrize("orig,new", RATE_PAIRS)
def test_compact_spans_cover_every_tap_and_fit(orig, new):
    k, w = sinc_resample_kernel(orig, new)
    k = k.reshape(k.shape[0], -1)
    total = 0
    for row in k:
        nz = row.nonzero().flatten()
        assert nz.numel() > 0
        f, l = int(nz.min()), int(nz.max())
        assert not row[:f].any() and not row[l + 1:].any()     # everything outside the span is an exact zero
        total += l - f + 1
    assert total * 8 + (2 * k.shape[0] + 1) * 4 <= TABLE_MAX_BYTES, (orig, new, total)


def test_near_coprime_pair_is_refused_with_its_size():
    with pytest.raises(ValueError, match="bytes"):
        Resample(16001, 16000)
    with pytest.raises(NotImplementedError):
        sinc_resample_kernel(44100, 16000, resampling_method="sinc_interp_kaiser")


@pytest.mark.parametrize("orig,new", RATE_PAIRS)
def test_output_length_matches_torchaudio(orig, new):
    rs = Resample(orig, new)
    g = math.gcd(orig, new)
    lens = list(range(0, 3000)) + [10 ** 6 + 7, 44100 * 3600 + 1, 2 ** 31 - 1]
    o, nn = orig // g, new // g
    for n in lens:
        # _apply_sinc_resample_kernel: conv1d yields (n // o + 1) frames of nn phases, sliced to the float32 target
        target = int(torch.ceil(torch.as_tensor(nn * n / o)).long())
        assert rs.output_length(n) == min(target, (n // o + 1) * nn), n
    for n in (1, 5, 441, 1777):
        assert CO.resample(torch.ones(n), orig, new).numel() == rs.output_length(n)
    assert Resample(16000, 16000).output_length(123) == 123


def _tool_keys(configs):
    """compute_cmvn_stats.py:109-116 restated."""
    feat_type = configs["dataset_conf"]["feats_type"]
    feat_dim = configs["dataset_conf"][f"{feat_type}_conf"]["num_mel_bins"]
    rr = configs["dataset_conf"]["resample_conf"]["resample_rate"] if "resample_conf" in configs["dataset_conf"] else 0
    return feat_type, feat_dim, rr


def test_from_config_reads_the_tools_keys():
    cfgs = [{"dataset_conf": {"feats_type": "fbank", "fbank_conf": {"num_mel_bins": 40}, "resample_conf":
                              {"resample_rate": 16000}}},
            {"dataset_conf": {"feats_type": "mfcc", "mfcc_conf": {"num_mel_bins": 80}}}]
    if have_reference():
        import glob
        import yaml
        for p in sorted(glob.glob(os.path.join(REFERENCE, "examples", "*", "s0", "conf", "*.yaml"))):
            with open(p) as f:
                cfgs.append(yaml.safe_load(f))
    legacy = 0
    for c in cfgs:
        try:
            want = _tool_keys(c)
        except KeyError:
            legacy += 1
            with pytest.raises(KeyError):
                CmvnStats.from_config(c)
            continue
        s = CmvnStats.from_config(c)
        assert (s.feat_type, s.feat_dim, s.resample_rate) == want
        assert s.frontend.feature_dim == want[1]
    assert legacy >= (1 if have_reference() else 0)
    with pytest.raises(KeyError):        # mdtc.yaml's layout
        CmvnStats.from_config({"dataset_conf": {"feature_extraction_conf": {"feature_type": "mfcc"}}})
    with pytest.raises(NotImplementedError):
        CmvnStats("fbank", 40, resample_rate=8000)
    with pytest.raises(ValueError):
        CmvnStats("spectrogram", 40)


def test_scp_segment_as_the_tool():
    assert scp_segment("/a/b.wav", 16000) == ("/a/b.wav", None, None)
    assert scp_segment(" /a/b.wav,0.13,0.81\n", 44100) == ("/a/b.wav", int(0.13 * 44100), int(0.81 * 44100))
    assert scp_segment("/a/b.wav,1,2.5", 8000) == ("/a/b.wav", 8000, 20000)
    for bad in ("/a/b.wav,1", "/a/b.wav,1,2,3"):
        with pytest.raises(ValueError):
            scp_segment(bad, 16000)
