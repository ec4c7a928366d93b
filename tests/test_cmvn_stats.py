"""Global CMVN statistics and resampling on the device (csrc/resample.cu, csrc/cmvn_stats.cu) against the golden of
the reference's tools/compute_cmvn_stats.py and the CPU oracle (oracle/kws_cmvn_oracle.py)."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import kws_cmvn_oracle as CO
from tests.conftest import ROOT, golden
from tests.test_cmvn_stats_host import golden_items
from wekws_b200 import CmvnStats, Resample, load_cmvn, resample, scp_segment, _native

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL_FEAT_MEAN = 1e-5          # tests/test_gpu_parity.py _check_feats: mean |feature error| of the Fbank kernel
TOL_MFCC_MEAN = 6e-4          # tests/test_gpu_parity.py _check_mfcc: the same for the MFCC epilogue
SRC_RATES = [r for r in CO.RATES if r != 16000]


def _check_resampled(out, x, orig, new, ta=None):
    """out: our row; x: its input.  Within 1 ulp of the float64 evaluation (plus the spread two double summation
    orders can have, 2^-50 sum |k| |x|), and at least as close to it as torchaudio's float32 conv1d."""
    if x.numel() == 0:                 # torchaudio raises on an empty waveform; the batch form gives an empty row
        assert out.size == 0
        return
    f64 = CO.resample(x.double(), orig, new, torch.float64).numpy()
    out = out.astype(np.float64)
    assert out.shape == f64.shape
    if not f64.size:
        return
    slack = 2.0 ** -50 * CO.resample_abs_bound(x, orig, new).numpy()
    ulp = np.spacing(np.abs(f64).astype(np.float32)).astype(np.float64)
    err = np.abs(out - f64)
    assert (err <= ulp + slack).all(), (orig, float((err / ulp).max()))
    if ta is None:
        ta = CO.resample(x.float(), orig, new).numpy()
    assert (err <= np.abs(ta.astype(np.float64) - f64) + 0.5 * ulp + slack).all()


@pytest.mark.parametrize("orig", SRC_RATES)
def test_resample_accuracy(orig):
    g = golden("cmvn_stats")
    rs = Resample(orig, 16000)
    x = torch.from_numpy(g[f"rs_in_{orig}"])
    for pcm in (x, x.float()):
        _check_resampled(rs(pcm.to(DEV)).cpu().numpy(), x.float(), orig, 16000, g[f"rs_ta_{orig}"])
    o = orig // math.gcd(orig, 16000)
    long = torch.from_numpy(CO.scripted_wave(orig + 1, 3 * o + 5 * 441 + 17))
    lens = [0, 1, max(1, o - 1), o, o + 1, 2345, long.numel()]
    batch = torch.zeros(len(lens), long.numel(), dtype=torch.int16)
    for b, n in enumerate(lens):
        batch[b, :n] = long[:n]
    for pcm in (batch, batch.float()):
        out = rs(pcm.to(DEV), torch.tensor(lens)).cpu().numpy()
        for b, n in enumerate(lens):
            m = rs.output_length(n)
            _check_resampled(out[b, :m], long[:n].float(), orig, 16000)
            assert not out[b, m:].any()


@pytest.mark.parametrize("N", [7001, 7008])      # 7008: 16-byte rows, the vector staging path; 7001: the scalar one
@pytest.mark.parametrize("orig,new", [(44100, 16000), (8000, 16000), (16000, 48000), (48000, 16000)])
def test_resample_layout(orig, new, N):
    rs = Resample(orig, new)
    torch.manual_seed(5)
    B = 9
    lens = [N, 0, 1, 400, 441, 3000, 6999, 5000, 17]
    x = (torch.randn(B, N) * 3000).round()
    for b, n in enumerate(lens):
        x[b, n:] = float("nan")                       # never read: past lens[b] counts as zeros
    out = rs(x.to(DEV), torch.tensor(lens)).cpu()
    assert out.shape == (B, rs.output_length(N))
    for b, n in enumerate(lens):
        m = rs.output_length(n)
        assert torch.isfinite(out[b]).all() and not out[b, m:].any()
        one = rs(x[b, :n].contiguous().to(DEV)).cpu() if n else torch.zeros(0)
        assert torch.equal(out[b, :m], one), b
        if n:
            clean = x[b, :n].nan_to_num(0.0)
            _check_resampled(out[b, :m].numpy(), clean, orig, new)
    # rows that start 2 bytes past an aligned address take the scalar staging path; they must agree bitwise with the
    # same rows at an aligned address (the vector path when N is a multiple of 8)
    xi = x.nan_to_num(0.0).to(torch.int16)
    wide = torch.zeros(B, N + 3, dtype=torch.int16)
    wide[:, 1:N + 1] = xi
    a = rs(xi.to(DEV), torch.tensor(lens)).cpu()
    s = rs(wide.to(DEV)[:, 1:N + 1], torch.tensor(lens)).cpu()
    assert torch.equal(a, s)
    assert resample(xi, orig, orig) is xi and Resample(orig, orig)(xi) is xi       # equal rates: the input itself


def _feed(stats, items, batch=None):
    """items [(waveform int16-scale float32 (N,), rate)] -> stats.update per run of equal rate (in order)."""
    i = 0
    while i < len(items):
        j = i
        while j < len(items) and items[j][1] == items[i][1] and (batch is None or j - i < batch):
            j += 1
        wavs = [w for w, _ in items[i:j]]
        n = max(w.numel() for w in wavs)
        pcm = torch.zeros(len(wavs), n)
        for b, w in enumerate(wavs):
            pcm[b, :w.numel()] = w
        stats.update(pcm.to(torch.int16).to(DEV), [w.numel() for w in wavs], items[i][1])
        i = j


def _sum_bound(truth_feats_abs2, frames, ref_err, tol_mean):
    """Per-dimension bound on |S_ours - S_f64|, _check_feats's rule carried over to the sums.  _check_feats accepts
    features whose mean |error| is tol_mean (TOL_FEAT_MEAN, or TOL_MFCC_MEAN in _check_mfcc), or, where the
    reference's own float32 error is larger, at most 1.5x the reference's.  A sum over `frames` rows then errs by at most frames * tol_mean for sum x, and for sum x^2
    (d(x^2) = 2 |x| dx) by tol_mean * sum 2 |x|; or by 1.5x the reference's own error of the same sum (its float32
    features and float32 accumulators)."""
    floor = np.stack([np.full(ref_err.shape[1], frames * tol_mean), tol_mean * truth_feats_abs2])
    return np.maximum(1.5 * ref_err, floor)


def _truth(items, ft, dim):
    """float64 evaluation of the whole chain: (frames, (2, D) sums, sum 2|x| per dimension)."""
    s = np.zeros((2, dim))
    a2 = np.zeros(dim)
    n = 0
    for w, r in items:
        x = CO.resample(w.double(), r, 16000, torch.float64) if r != 16000 else w.double()
        f = CO.features(x, ft, dim, 16000, torch.float64).numpy()
        s[0] += f.sum(0)
        s[1] += (f * f).sum(0)
        a2 += 2 * np.abs(f).sum(0)
        n += f.shape[0]
    return n, s, a2


@pytest.fixture(scope="module")
def truth():
    cache = {}

    def get(ft, dim):
        if (ft, dim) not in cache:
            cache[(ft, dim)] = _truth(golden_items(), ft, dim)
        return cache[(ft, dim)]
    return get


@pytest.mark.parametrize("case", ["fbank40", "fbank80", "mfcc80"])
def test_stats_match_reference_golden(case, truth):
    g = golden("cmvn_stats")
    ft, dim = ("mfcc", 80) if case == "mfcc80" else ("fbank", int(case[5:]))
    ref = json.loads(str(g[f"{case}_json"]))
    stats = CmvnStats(ft, dim, resample_rate=16000)
    items = sorted(golden_items(), key=lambda it: it[1])         # one batch per rate
    _feed(stats, items)
    n, s64, a2 = truth(ft, dim)
    assert stats.frame_num == ref["frame_num"] == n
    ours = np.stack([stats.mean_stat.numpy(), stats.var_stat.numpy()])
    ref_s = np.array([ref["mean_stat"], ref["var_stat"]], dtype=np.float64)
    bound = _sum_bound(a2, n, np.abs(ref_s - s64), TOL_MFCC_MEAN if ft == "mfcc" else TOL_FEAT_MEAN)
    assert (np.abs(ours - s64) <= bound).all(), float((np.abs(ours - s64) / bound).max())
    # the loaded CMVN: mean = S / n, var = Q / n - mean^2, istd = var^-1/2; propagate the same bound
    js = json.loads(stats.to_json())
    assert set(js) == {"mean_stat", "var_stat", "frame_num"} and js["frame_num"] == n
    d = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"cmvn_{os.getpid()}_{case}")
    stats.write(d + "_ours")
    with open(d + "_ref", "w") as f:
        f.write(str(g[f"{case}_json"]))
    m_o, i_o = load_cmvn(d + "_ours")
    m_r, i_r = load_cmvn(d + "_ref")
    os.remove(d + "_ours")
    os.remove(d + "_ref")
    mu = s64[0] / n
    var = s64[1] / n - mu * mu
    b_mean = 2 * bound[0] / n
    b_var = 2 * bound[1] / n + 2 * np.abs(mu) * b_mean + b_mean ** 2
    b_istd = 0.5 * var ** -1.5 * b_var * 1.01
    assert (np.abs(m_o - m_r) <= b_mean).all() and (np.abs(i_o - i_r) <= b_istd).all()


def test_stats_deterministic_across_batching():
    items = []
    for i in range(60):                # 44.1 kHz utterances of 0.15 to 1.0 s
        n = int(44100 * (0.15 + 0.25 * (i % 2) + 0.01 * i))
        items.append((torch.from_numpy(CO.scripted_wave(300 + i, n).astype(np.float32)), 44100))
    runs = []
    for batch in (60, 20, 60):
        st = CmvnStats("fbank", 80, resample_rate=16000)
        _feed(st, items, batch)
        runs.append((st.frame_num, st.mean_stat, st.var_stat))
    for r in runs[1:]:
        assert r[0] == runs[0][0] and torch.equal(r[1], runs[0][1]) and torch.equal(r[2], runs[0][2])


def test_stats_scale_44k():
    g = torch.Generator().manual_seed(11)
    B = 512
    lens = torch.randint(int(0.5 * 44100), 10 * 44100 + 1, (B,), generator=g)
    lens[0] = 10 * 44100
    pcm = (torch.randn(B, int(lens.max()), generator=g) * 2000).round().to(torch.int16)
    st = CmvnStats("fbank", 80, resample_rate=16000)
    st.update(pcm.to(DEV), lens, 44100)
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    items = [(pcm[b, :int(lens[b])].float(), 44100) for b in range(B)]
    n, _, _, s64 = CO.collate(items, "fbank", 80, 16000)
    assert st.frame_num == n
    # both feature sets are within the Fbank gate of the truth, so their sums differ by at most twice _sum_bound's
    # floor; a log-mel of int16-scale audio has |x| < 40, so sum 2|x| over n frames is below 80 n
    ours = np.stack([st.mean_stat.numpy(), st.var_stat.numpy()])
    bound = 2 * _sum_bound(np.full(80, 80.0 * n), n, np.zeros((2, 80)), TOL_FEAT_MEAN)
    assert (np.abs(ours - s64.numpy()) <= bound).all()


def test_handles_survive_later_creates():
    """The shared-memory limit is a property of the kernel function: a handle created later with a smaller table
    must not break the forward of an earlier one with a larger table."""
    x = torch.from_numpy(CO.scripted_wave(21, 3 * 44100)).to(DEV)
    a = Resample(44100, 16000)
    ya = a(x)
    for orig in (48000, 8000):
        y = Resample(orig, 16000)(x)
        assert y.numel() > 0
        assert torch.equal(a(x), ya)
    _check_resampled(ya.cpu().numpy(), x.cpu().float(), 44100, 16000)


def test_stats_interleaved_rates():
    """A feed whose rates alternate (44.1, 48, 44.1, 8 kHz) reuses each rate's cached resampler after others were
    built; it matches the oracle as the CLI does."""
    items = []
    for i, rate in enumerate((44100, 48000, 44100, 8000, 48000)):
        for j in range(3):
            items.append((torch.from_numpy(CO.scripted_wave(700 + 3 * i + j, int(rate * (0.5 + 0.1 * j))).astype(
                np.float32)), rate))
    st = CmvnStats("fbank", 40, resample_rate=16000)
    _feed(st, items)
    n, _, _, s64 = CO.collate(items, "fbank", 40, 16000)
    assert st.frame_num == n
    ours = np.stack([st.mean_stat.numpy(), st.var_stat.numpy()])
    assert (np.abs(ours - s64.numpy()) <= 2 * _sum_bound(np.full(40, 80.0 * n), n, np.zeros((2, 40)),
                                                        TOL_FEAT_MEAN)).all()


def test_launch_counts():
    st = CmvnStats("mfcc", 80, resample_rate=16000)
    pcm = torch.from_numpy(CO.scripted_wave(3, 3 * 48000)).repeat(3, 1).to(DEV)
    n0 = _native.launch_count()
    st.update(pcm, [3 * 48000, 48000, 20000], 48000)
    assert _native.launch_count() - n0 == 4                     # resample 1, fbank 1, statistics 2
    n0 = _native.launch_count()
    st.update(pcm, None, 16000)
    assert _native.launch_count() - n0 == 3
    assert st.frame_num > 0


def test_refusals():
    st = CmvnStats("fbank", 40, resample_rate=16000)
    pcm = torch.zeros(3, 1000, dtype=torch.int16, device=DEV)
    with pytest.raises(ValueError, match="utterance 1"):
        st.update(pcm, [1000, 300, 1000], 16000)                 # kaldi.fbank asserts on < 400 samples
    with pytest.raises(ValueError, match="utterance 2"):
        st.update(pcm, [1000, 1000, 199], 8000)                  # 199 samples at 8 kHz -> 398 at 16 kHz
    with pytest.raises(NotImplementedError):
        CmvnStats("fbank", 40).update(pcm, None, 8000)           # no resample_conf, 8 kHz audio
    with pytest.raises(RuntimeError):
        st.update(pcm.cpu(), None, 16000)
    assert st.frame_num == 0
    with pytest.raises(ValueError, match="bytes"):
        Resample(16001, 16000)
    with pytest.raises(RuntimeError, match="bytes"):             # the compact table does not fit shared memory
        Resample(4001, 4000)(torch.zeros(8000, device=DEV))
    with pytest.raises(RuntimeError):
        Resample(44100, 16000)(torch.zeros(100))


def test_cli_end_to_end(tmp_path):
    from scipy.io import wavfile
    lines, items = [], []
    for i, rate in enumerate((8000, 16000, 22050, 44100, 48000)):
        for j, seg in enumerate((None, (0.11, 0.74))):
            x = CO.scripted_wave(50 + 2 * i + j, int(rate * (0.9 + 0.05 * i)))
            p = tmp_path / f"u{i}{j}.wav"
            if j == 0 and i % 2:
                wavfile.write(p, rate, x.astype(np.float32) / 32768)     # float32 WAV
            else:
                wavfile.write(p, rate, x)
            value = str(p) if seg is None else f"{p},{seg[0]},{seg[1]}"
            lines.append(f"u{i}{j} {value}")
            _, s, e = scp_segment(value, rate)
            items.append((torch.from_numpy((x if s is None else x[s:e]).astype(np.float32)), rate))
    (tmp_path / "wav.scp").write_text("\n".join(lines) + "\n")
    (tmp_path / "train.yaml").write_text("dataset_conf:\n  resample_conf:\n    resample_rate: 16000\n"
                                         "  feats_type: fbank\n  fbank_conf:\n    num_mel_bins: 40\n")
    out = tmp_path / "global_cmvn"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "scripts", "compute_cmvn_stats.py"), "--num_workers", "16",
                        "--train_config", str(tmp_path / "train.yaml"), "--in_scp", str(tmp_path / "wav.scp"),
                        "--out_cmvn", str(out), "--batch", "3"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    js = json.loads(out.read_text())
    n, m32, v32, s64 = CO.collate(items, "fbank", 40, 16000)
    assert js["frame_num"] == n
    a2 = 2 * 40.0 * n
    ours = np.array([js["mean_stat"], js["var_stat"]])
    bound = np.stack([np.full(40, 2 * n * TOL_FEAT_MEAN), np.full(40, 2 * TOL_FEAT_MEAN * a2)])
    assert (np.abs(ours - s64.numpy()) <= bound).all()
    mean, istd = load_cmvn(str(out))
    assert mean.shape == (40,) and np.isfinite(istd).all() and (istd > 0).all()
    from wekws_b200 import init_model, model_config
    cfg = dict(model_config("ds_tcn"), input_dim=40, cmvn={"norm_var": True, "cmvn_file": str(out)})
    m = init_model(cfg)
    assert torch.allclose(m.global_cmvn.mean, torch.from_numpy(mean).float())
