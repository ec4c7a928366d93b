"""CPU oracle for the WeKws streaming keyword-spotting forward path.

TEST INFRASTRUCTURE ONLY.  Nothing in ``wekws_b200/`` imports this module; only
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py`` (its ``cpu_baseline`` leg
and ``--impl reference`` arm) may.  It is the checker, never the product.

It restates, op for op and in fp32 on the CPU, what the reference computes:

* ``fbank``           -> torchaudio.compliance.kaldi.fbank as called from
                         wekws/dataset/processor.py:173-203 and
                         wekws/bin/stream_kws_ctc.py:354-360
                         (torchaudio 2.11.0 kaldi.py:44-83 framing, :154-217
                         window, :436-511 mel banks, :616-633 spectrum/mel/log)
* ``global_cmvn``     -> wekws/model/cmvn.py:37-48
* ``load_cmvn_json``  -> wekws/utils/cmvn.py:23-45
* ``kws_forward``     -> wekws/model/kws_model.py:65-76 which composes
                         subsampling.py:53-57, mdtc.py:95-121/181-198/242-276,
                         tcn.py:35-61/75-84/101-114/139-166, torch.nn.GRU
                         (kws_model.py:130-133), classifier.py:63-67 and the
                         activation chosen at kws_model.py:196-210.

The model is described by the ``model`` section of a reference yaml config (plus
``input_dim``/``output_dim`` as wekws/bin/train.py:134-146 injects them) and a
reference-format ``state_dict``.  The same ATen ops the reference dispatches to
(conv1d, batch_norm with running stats, linear, gru) are used on purpose, so
that timing this module on host cores is a fair stand-in for the reference's
own CPU path on a machine where /root/reference does not exist.

Parity pinning: ``tests/test_oracle_pinned.py`` checks every function here
against golden vectors produced by the real reference (``oracle/make_golden.py``
imports /root/reference and torchaudio and writes ``tests/golden/*.npz``), and,
when /root/reference is present, against the live reference.
"""
from __future__ import annotations

import json
import math
from typing import Dict, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor

EPS = float(torch.finfo(torch.float32).eps)  # kaldi.py:21
BN_EPS = 1e-5  # torch.nn.BatchNorm1d default, used by every BN in mdtc.py / tcn.py


# --------------------------------------------------------------------------- Fbank
def povey_window(n: int, dtype=torch.float32) -> Tensor:
    """kaldi.py:98-100: hann(n, periodic=False) ** 0.85 (fp32 in the reference)."""
    return torch.hann_window(n, periodic=False, dtype=dtype).pow(0.85)


def hamming_window(n: int, dtype=torch.float32) -> Tensor:
    """kaldi.py:96-97 / runtime/core/frontend/fbank.h:90-96."""
    return torch.hamming_window(n, periodic=False, alpha=0.54, beta=0.46, dtype=dtype)


def mel_scale(f: Tensor) -> Tensor:
    return 1127.0 * (1.0 + f / 700.0).log()  # kaldi.py:330-331


def mel_banks(num_bins: int, n_fft: int, sample_rate: float,
              low_freq: float = 20.0, high_freq: float = 0.0, dtype=torch.float32) -> Tensor:
    """kaldi.py:436-511 with vtln_warp == 1.0.  Returns (num_bins, n_fft//2 + 1);
    the extra last column (Nyquist) is the zero pad of kaldi.py:627."""
    num_fft_bins = n_fft // 2
    nyquist = 0.5 * sample_rate
    if high_freq <= 0.0:
        high_freq += nyquist
    fft_bin_width = sample_rate / n_fft
    mel_low = 1127.0 * math.log(1.0 + low_freq / 700.0)
    mel_high = 1127.0 * math.log(1.0 + high_freq / 700.0)
    delta = (mel_high - mel_low) / (num_bins + 1)
    b = torch.arange(num_bins).unsqueeze(1)
    left = mel_low + b * delta
    center = mel_low + (b + 1.0) * delta
    right = mel_low + (b + 2.0) * delta
    mel = mel_scale(fft_bin_width * torch.arange(num_fft_bins, dtype=dtype)).unsqueeze(0)
    up = (mel - left) / (center - left)
    down = (right - mel) / (right - center)
    bins = torch.max(torch.zeros(1, dtype=dtype), torch.min(up, down))
    return F.pad(bins, (0, 1), mode="constant", value=0.0)


def num_frames(num_samples: int, frame_len: int = 400, frame_shift: int = 160) -> int:
    """snip_edges framing, kaldi.py:66-70."""
    if num_samples < frame_len:
        return 0
    return 1 + (num_samples - frame_len) // frame_shift


def feature_window(window_type: str, n: int, dtype=torch.float32) -> Tensor:
    """kaldi.py:86-113 without blackman: povey, hanning, hamming or rectangular."""
    if window_type == "povey":
        return povey_window(n, dtype)
    if window_type == "hanning":
        return torch.hann_window(n, periodic=False, dtype=dtype)
    if window_type == "hamming":
        return hamming_window(n, dtype)
    if window_type == "rectangular":
        return torch.ones(n, dtype=dtype)
    raise ValueError("Invalid window type " + window_type)


def fbank(waveform: Tensor, num_mel_bins: int = 80, frame_length: float = 25.0,
          frame_shift: float = 10.0, sample_frequency: float = 16000.0,
          window_type: str = "povey", preemphasis: float = 0.97, dtype=torch.float32,
          remove_dc_offset: bool = True, low_freq: float = 20.0, high_freq: float = 0.0) -> Tensor:
    """Kaldi log-mel filterbank of one waveform (N,) in int16-scale floats, with
    dither=0, energy_floor=0 and the rest of kaldi.fbank's options at their defaults
    unless given here.  Returns (m, num_mel_bins).  dtype=float64 evaluates the same
    formulas in double (the 'exact arithmetic' yardstick tests use to rank fp32
    implementations)."""
    wav = waveform.to(dtype).reshape(-1)
    win = int(sample_frequency * frame_length * 0.001)
    shift = int(sample_frequency * frame_shift * 0.001)
    n_fft = 1 if win == 0 else 2 ** (win - 1).bit_length()
    m = num_frames(wav.numel(), win, shift)
    if m == 0:
        return torch.empty(0, num_mel_bins)
    frames = wav.as_strided((m, win), (shift, 1))                         # kaldi.py:82-83
    if remove_dc_offset:
        frames = frames - frames.mean(dim=1, keepdim=True)                # :183-186
    if preemphasis != 0.0:
        prev = F.pad(frames.unsqueeze(0), (1, 0), mode="replicate").squeeze(0)[:, :-1]
        frames = frames - preemphasis * prev                              # :193-198
    frames = frames * feature_window(window_type, win, dtype).unsqueeze(0)   # :201-204
    frames = F.pad(frames, (0, n_fft - win))                              # :207-211
    spec = torch.fft.rfft(frames).abs().pow(2.0)                          # :616-618
    mel = mel_banks(num_mel_bins, n_fft, sample_frequency, low_freq, high_freq, dtype=dtype)   # :621-627
    e = torch.mm(spec, mel.T)                                             # :630
    return torch.max(e, torch.tensor(EPS, dtype=dtype)).log()             # :633


def dct_matrix(num_ceps: int, num_mel_bins: int, dtype=torch.float32) -> Tensor:
    """(num_mel_bins, num_ceps): torchaudio kaldi.py _get_dct_matrix = functional.create_dct(n, n, 'ortho')
    with column 0 set to sqrt(1/n), first num_ceps columns."""
    n = torch.arange(float(num_mel_bins), dtype=dtype)
    k = torch.arange(float(num_mel_bins), dtype=dtype).unsqueeze(1)
    dct = torch.cos(math.pi / float(num_mel_bins) * (n + 0.5) * k)
    dct[0] *= 1.0 / math.sqrt(2.0)
    dct *= math.sqrt(2.0 / float(num_mel_bins))
    dct = dct.t().contiguous()
    dct[:, 0] = math.sqrt(1 / float(num_mel_bins))
    return dct[:, :num_ceps]


def mfcc(waveform: Tensor, num_ceps: int = 80, num_mel_bins: int = 80, cepstral_lifter: float = 22.0,
         frame_length: float = 25.0, frame_shift: float = 10.0, sample_frequency: float = 16000.0,
         window_type: str = "povey", dtype=torch.float32, preemphasis: float = 0.97,
         remove_dc_offset: bool = True, low_freq: float = 20.0, high_freq: float = 0.0) -> Tensor:
    """Kaldi MFCC of one waveform with the arguments the reference passes (wekws/dataset/processor.py:157-166:
    kaldi.mfcc(num_ceps, num_mel_bins, frame_length, frame_shift, dither=0, energy_floor=0, sample_frequency);
    use_energy False, htk_compat False, subtract_mean False by default), plus the front-end options of ``fbank``:
    log-mel fbank -> matmul with the DCT matrix -> cepstral lifter, none when cepstral_lifter is 0 (torchaudio
    kaldi.py mfcc body).  Returns (m, num_ceps)."""
    assert num_ceps <= num_mel_bins
    f = fbank(waveform, num_mel_bins, frame_length, frame_shift, sample_frequency, window_type, preemphasis, dtype,
              remove_dc_offset, low_freq, high_freq)
    if f.shape[0] == 0:
        return torch.empty(0, num_ceps)
    out = f.matmul(dct_matrix(num_ceps, num_mel_bins, dtype))
    if cepstral_lifter != 0.0:
        i = torch.arange(num_ceps)
        out = out * (1.0 + 0.5 * cepstral_lifter * torch.sin(math.pi * i / cepstral_lifter)).to(dtype).unsqueeze(0)
    return out


# ---------------------------------------------------------------------------- CMVN
def load_cmvn_json(path: str) -> Tuple[Tensor, Tensor]:
    """wekws/utils/cmvn.py:23-45, then the .float() of kws_model.py:104-108."""
    with open(path) as f:
        st = json.load(f)
    n = st["frame_num"]
    mean, istd = [], []
    for s, v in zip(st["mean_stat"], st["var_stat"]):
        mu = s / n
        var = v / n - mu * mu
        if var < 1.0e-20:
            var = 1.0e-20
        mean.append(mu)
        istd.append(1.0 / math.sqrt(var))
    return (torch.tensor(mean, dtype=torch.float64).float(),
            torch.tensor(istd, dtype=torch.float64).float())


def global_cmvn(x: Tensor, mean: Tensor, istd: Tensor, norm_var: bool = True) -> Tensor:
    x = x - mean
    if norm_var:
        x = x * istd
    return x


# --------------------------------------------------------------------------- model
def _bn(x: Tensor, sd: Dict[str, Tensor], p: str) -> Tensor:
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"],
                        sd[p + ".weight"], sd[p + ".bias"], False, 0.0, BN_EPS)


def _cat_cache(x: Tensor, cache: Optional[Tensor], pad: int) -> Tuple[Tensor, Tensor]:
    """mdtc.py:108-113 == tcn.py:49-54."""
    if cache is None:
        y = F.pad(x, (pad, 0), value=0.0)
    else:
        y = torch.cat((cache, x), dim=2)
    return y, y[:, :, -pad:]


def _mdtc_block(x, cache, sd, p, k, d):
    """mdtc.py:95-121 (TCNBlock) around mdtc.py:55-59 (DSDilatedConv1d)."""
    C = x.size(1)
    y, new_cache = _cat_cache(x, cache, d * (k - 1))
    o = F.conv1d(y, sd[p + ".conv1.conv.weight"], sd[p + ".conv1.conv.bias"], dilation=d, groups=C)
    o = _bn(o, sd, p + ".conv1.bn")
    o = F.conv1d(o, sd[p + ".conv1.pointwise.weight"], sd[p + ".conv1.pointwise.bias"])
    o = F.relu(_bn(o, sd, p + ".bn1"))
    o = _bn(F.conv1d(o, sd[p + ".conv2.weight"], sd[p + ".conv2.bias"]), sd, p + ".bn2")
    return F.relu(o + x), new_cache


def mdtc_layout(bb: dict):
    """(prefix, dilation) of the 1 + num_stack*stack_size blocks in cache order
    (mdtc.py:151-156, :236-237, :251-268)."""
    blocks = [("backbone.preprocessor", 1)]
    for s in range(bb["num_stack"]):
        for l in range(bb["stack_size"]):
            blocks.append((f"backbone.blocks.{s}.res_blocks.{l}", 2 ** l))
    return blocks


def _mdtc(x, cache, sd, bb):
    k = bb["kernel_size"]
    x = x.transpose(1, 2)
    off, caches, outs = 0, [], []
    for i, (p, d) in enumerate(mdtc_layout(bb)):
        pad = d * (k - 1)
        c_in = None if cache is None else cache[:, :, off:off + pad]
        x, c = _mdtc_block(x, c_in, sd, p, k, d)
        caches.append(c)
        off += pad
        if i > 0 and i % bb["stack_size"] == 0:
            outs.append(x)                                   # mdtc.py:266
    y = torch.zeros_like(outs[-1])
    for o in outs:
        y = y + o                                            # mdtc.py:270-273
    return y.transpose(1, 2), torch.cat(caches, dim=2)


def _tcn(x, cache, sd, bb):
    k = bb.get("kernel_size", 8)
    ds = bb.get("ds", False)
    x = x.transpose(1, 2)
    C = x.size(1)
    off, caches = 0, []
    for i in range(bb["num_layers"]):
        d = 2 ** i
        pad = (k - 1) * d
        p = f"backbone.network.{i}.cnn"
        c_in = None if cache is None else cache[:, :, off:off + pad]
        y, c = _cat_cache(x, c_in, pad)
        if ds:                                               # tcn.py:101-114
            y = F.relu(_bn(F.conv1d(y, sd[p + ".0.weight"], sd[p + ".0.bias"], dilation=d, groups=C), sd, p + ".1"))
            y = F.relu(_bn(F.conv1d(y, sd[p + ".3.weight"], sd[p + ".3.bias"]), sd, p + ".4"))
        else:                                                # tcn.py:75-84
            y = F.relu(_bn(F.conv1d(y, sd[p + ".0.weight"], sd[p + ".0.bias"], dilation=d), sd, p + ".1"))
        x = y + x                                            # tcn.py:60
        caches.append(c)
        off += pad
    return x.transpose(1, 2), torch.cat(caches, dim=2)


_GRU_CACHE: dict = {}


def _gru(x, cache, sd, bb, hdim):
    """torch.nn.GRU(hdim, hdim, num_layers, batch_first=True), kws_model.py:130-133.
    An empty cache raises in the reference (SURVEY: 'Expected hidden size ...');
    start-of-stream therefore means an explicit zero h0 here."""
    L = bb["num_layers"]
    dtype = sd["backbone.weight_ih_l0"].dtype                  # float64 state dicts give a float64 GRU
    key = (id(sd), L, hdim, dtype)
    g = _GRU_CACHE.get(key)
    if g is None:
        g = torch.nn.GRU(hdim, hdim, num_layers=L, batch_first=True, dtype=dtype)
        with torch.no_grad():
            for n, p in g.named_parameters():
                p.copy_(sd["backbone." + n])
        g.eval()
        _GRU_CACHE.clear()
        _GRU_CACHE[key] = g
    if cache is None:
        cache = x.new_zeros(L, x.size(0), hdim)
    with torch.no_grad():
        return g(x, cache)


def _fsmn(x, cache, sd, bb):
    """FSMN backbone (wekws/model/fsmn.py:401-495; SURVEY 8f-4 -- oracle only, no product kernel yet).
    in_linear1 -> in_linear2 -> ReLU -> num_layers x [LinearTransform (no bias) -> FSMNBlock -> AffineTransform ->
    ReLU] -> out_linear1 -> out_linear2.  FSMNBlock (fsmn.py:173-253): with p = cat(cache, h) along time
    (cache = (lorder-1) lstride + rorder rstride columns, zeros at the start of a stream),
        out[t] = p[t + (lorder-1) lstride] + sum_i wl[i] p[t + i lstride] + sum_j wr[j] p[t + (lorder-1) lstride + (j+1) rstride]
    i.e. the output is delayed by rorder*rstride frames; new cache = last columns of p.  The 4-D cache is
    (B, proj_dim, cache_len, num_layers)."""
    L, lo, ro = bb["num_layers"], bb["left_order"], bb["right_order"]
    # the reference builds every block with strides (1, 1) whatever the config says (_build_repeats, fsmn.py:384-391
    # passes the literals 1, 1); left_stride / right_stride only enter FSMN.padding, which the forward never uses
    ls, rs = 1, 1
    assert ro >= 1, "the reference's FSMNBlock slices x_pad[:, :, :-rorder*rstride] and breaks for right_order = 0"
    pad = (lo - 1) * ls + ro * rs
    B, T, _ = x.shape
    h = F.linear(x, sd["backbone.in_linear1.linear.weight"], sd["backbone.in_linear1.linear.bias"])
    h = F.relu(F.linear(h, sd["backbone.in_linear2.linear.weight"], sd["backbone.in_linear2.linear.bias"]))
    new_caches = []
    for l in range(L):
        pre = f"backbone.fsmn.{l}."
        p = F.linear(h, sd[pre + "0.linear.weight"])                               # (B, T, proj)
        pt = p.transpose(1, 2)                                                      # (B, proj, T)
        c = pt.new_zeros(B, pt.size(1), pad) if cache is None else cache[:, :, :, l]
        cat = torch.cat((c, pt), dim=2)                                             # fsmn.py:226-231
        new_caches.append(cat[:, :, -pad:] if pad > 0 else cat[:, :, :0])           # :232-233
        wl = sd[pre + "1.conv_left.weight"].reshape(-1, lo)                          # (proj, lorder)
        out = cat[:, :, (lo - 1) * ls:(lo - 1) * ls + T].clone()                     # :238-239
        for i in range(lo):
            out = out + wl[:, i].reshape(1, -1, 1) * cat[:, :, i * ls:i * ls + T]    # :235-237 (valid conv, dilation ls)
        if ro > 0:
            wr = sd[pre + "1.conv_right.weight"].reshape(-1, ro)
            base = (lo - 1) * ls + rs                                                # :241-248
            for j in range(ro):
                out = out + wr[:, j].reshape(1, -1, 1) * cat[:, :, base + j * rs:base + j * rs + T]
        h = F.relu(F.linear(out.transpose(1, 2), sd[pre + "2.linear.weight"], sd[pre + "2.linear.bias"]))
    h = F.linear(h, sd["backbone.out_linear1.linear.weight"], sd["backbone.out_linear1.linear.bias"])
    h = F.linear(h, sd["backbone.out_linear2.linear.weight"], sd["backbone.out_linear2.linear.bias"])
    return h, torch.stack(new_caches, dim=3)


def backbone_padding(cfg: dict) -> int:
    bb = cfg["backbone"]
    if bb["type"] == "mdtc":
        k = bb["kernel_size"]
        return sum(d * (k - 1) for _, d in mdtc_layout(bb))
    if bb["type"] == "tcn":
        k = bb.get("kernel_size", 8)
        return sum((k - 1) * 2 ** i for i in range(bb["num_layers"]))
    return 0


@torch.no_grad()
def kws_forward(sd: Dict[str, Tensor], cfg: dict, feats: Tensor,
                cache: Optional[Tensor] = None, softmax: bool = False) -> Tuple[Tensor, Tensor]:
    """KWSModel.forward (kws_model.py:65-76); ``softmax=True`` is forward_softmax (:78-90).
    ``cache`` None or of size(0)==0 means start of stream."""
    if cache is not None and cache.numel() == 0:
        cache = None
    x = feats
    if "global_cmvn.mean" in sd:
        x = global_cmvn(x, sd["global_cmvn.mean"], sd["global_cmvn.istd"],
                        cfg.get("cmvn", {}).get("norm_var", True))
    bb = cfg["backbone"]
    if bb["type"] == "fsmn":      # preprocessing 'none' (NoSubsampling), classifier 'identity' (kws_model.py:121-122,191)
        x, new_cache = _fsmn(x, cache, sd, bb)
        if cfg.get("activation", {}).get("type", "sigmoid") != "identity":
            x = torch.sigmoid(x)
        return (x.softmax(2) if softmax else x), new_cache
    x = F.relu(F.linear(x, sd["preprocessing.out.0.weight"], sd["preprocessing.out.0.bias"]))
    if bb["type"] == "mdtc":
        x, new_cache = _mdtc(x, cache, sd, bb)
    elif bb["type"] == "tcn":
        x, new_cache = _tcn(x, cache, sd, bb)
    elif bb["type"] == "gru":
        x, new_cache = _gru(x, cache, sd, bb, cfg["hidden_dim"])
    else:
        raise ValueError("oracle: unsupported backbone " + str(bb["type"]))
    x = F.linear(x, sd["classifier.linear.weight"], sd["classifier.linear.bias"])
    if cfg.get("activation", {}).get("type", "sigmoid") != "identity":
        x = torch.sigmoid(x)
    if softmax:
        x = x.softmax(2)
    return x, new_cache


# ---------------------------------------------------------------------------- detection statistics
def det_stats(post: Tensor, lengths, step: float = 0.01, window_shift: int = 50):
    """Pure-Python restatement of wekws/bin/score.py:128-137 (scores written as '{:.6f}') followed by
    wekws/bin/compute_det.py:76-105 (threshold sweep; triggers counted left to right with a window_shift skip).
    post (B, T, K).  Returns (thresholds list, max_score [B][K], triggers [B][K][n])."""
    B, T, K = post.shape
    thresholds, threshold = [], 0.0
    while threshold <= 1.0:                                   # compute_det.py:79-105
        thresholds.append(threshold)
        threshold += step
    max_score = [[None] * K for _ in range(B)]
    triggers = [[None] * K for _ in range(B)]
    for b in range(B):
        n = T if lengths is None else int(lengths[b])
        for k in range(K):
            text = ' '.join(['{:.6f}'.format(x) for x in post[b, :n, k].tolist()])      # score.py:133-135
            score_list = list(map(float, text.split()))                                 # compute_det.py:30
            max_score[b][k] = max(score_list) if score_list else float('-inf')         # :83
            row = []
            for th in thresholds:
                count, i = 0, 0
                while i < len(score_list):                                              # :91-97
                    if score_list[i] >= th:
                        count += 1
                        i += window_shift
                    else:
                        i += 1
                row.append(count)
            triggers[b][k] = row
    return thresholds, max_score, triggers


def det_curve_text(thresholds, max_score, triggers, kinds, durations, k: int) -> str:
    """The stats file wekws/bin/compute_det.py:76-105 writes for keyword index k, from det_stats outputs:
    kinds[b] == k marks keyword utterances (compute_det.py:44-46), every other utterance is filler and adds its
    duration (:47-49).  Pinned by tests/golden/det_stats.npz, which the reference tool itself wrote
    (oracle/make_det_golden.py)."""
    B = len(kinds)
    kw = [b for b in range(B) if kinds[b] == k]
    fil = [b for b in range(B) if kinds[b] != k]
    filler_duration = 0.0
    for b in fil:
        filler_duration += float(durations[b])
    lines = []
    false_reject_rate = false_alarm_per_hour = None
    for i, threshold in enumerate(thresholds):
        num_false_reject = sum(1 for b in kw if float(max_score[b][k]) < threshold)          # :81-85
        num_false_alarm = sum(triggers[b][k][i] for b in fil)                                # :86-97
        if len(kw) != 0:
            false_reject_rate = num_false_reject / len(kw)
        num_false_alarm = max(num_false_alarm, 1e-6)
        if filler_duration != 0:
            false_alarm_per_hour = num_false_alarm / (filler_duration / 3600.0)
        lines.append('{:.6f} {:.6f} {:.6f}\n'.format(threshold, false_alarm_per_hour, false_reject_rate))
    return ''.join(lines)


# ---------------------------------------------------------------------------- input transforms of the CTC recipes
def context_expansion(feats: Tensor, left: int = 1, right: int = 1) -> Tensor:
    """wekws/dataset/processor.py:267-296 for one utterance (T, D) -> (T - right, D * (left + right + 1)): roll-based
    stacking of lags -left..right, first frame replicated into the left margin (:288-292), last `right` frames dropped
    (:294).  Pinned by tests/golden/context.npz (made by running the reference function itself)."""
    T, D = feats.shape
    out = torch.zeros(T, D * (left + right + 1), dtype=torch.float32)
    index = 0
    for lag in range(-left, right + 1):
        out[:, index:index + D] = torch.roll(feats, -lag, 0)
        index += D
    for idx in range(left):
        for cpx in range(left - idx):
            out[idx, cpx * D:(cpx + 1) * D] = out[left, :D]
    return out[:T - right]


def frame_skip(feats: Tensor, skip_rate: int = 1) -> Tensor:
    """wekws/dataset/processor.py:299-312."""
    return feats[::skip_rate, :]


# ---------------------------------------------------------------------------- CTC prefix beam search + keyword look-up
def ctc_prefix_beam_search(probs: Tensor, keywords_tokenset=None, score_beam_size: int = 3, path_beam_size: int = 20,
                           cur_hyps=None, frame_offset: int = 0, frame_stride: int = 1):
    """Restatement of wekws/model/loss.py:206-312 (same statements in the same order, incl. the shared node dicts), with
    the streaming twin's extras (wekws/bin/stream_kws_ctc.py:124-215,400-409): hypotheses can be carried in and frames
    are numbered frame_offset + t * frame_stride.  probs (T, V).  Returns the pruned cur_hyps list
    [(prefix, (pb, pnb, nodes))]; hyps_of() gives loss.py's return value.  Pinned by tests/golden/ctc.npz."""
    import math
    from collections import defaultdict
    if cur_hyps is None:
        cur_hyps = [(tuple(), (1.0, 0.0, []))]
    for row in range(probs.size(0)):
        t = frame_offset + row * frame_stride
        p = probs[row]
        next_hyps = defaultdict(lambda: (0.0, 0.0, []))
        top_k_probs, top_k_index = p.topk(score_beam_size)
        filter_index = []
        for prob, idx in zip(top_k_probs.tolist(), top_k_index.tolist()):
            if prob > 0.05 and (keywords_tokenset is None or idx in keywords_tokenset):
                filter_index.append(idx)
        if len(filter_index) == 0:
            continue
        for s in filter_index:
            ps = p[s].item()
            for prefix, (pb, pnb, cur_nodes) in cur_hyps:
                last = prefix[-1] if len(prefix) > 0 else None
                if s == 0:
                    n_pb, n_pnb, nodes = next_hyps[prefix]
                    n_pb = n_pb + pb * ps + pnb * ps
                    nodes = cur_nodes.copy()
                    next_hyps[prefix] = (n_pb, n_pnb, nodes)
                elif s == last:
                    if not math.isclose(pnb, 0.0, abs_tol=0.000001):
                        n_pb, n_pnb, nodes = next_hyps[prefix]
                        n_pnb = n_pnb + pnb * ps
                        nodes = cur_nodes.copy()
                        if ps > nodes[-1]['prob']:
                            nodes[-1]['prob'] = ps
                            nodes[-1]['frame'] = t
                        next_hyps[prefix] = (n_pb, n_pnb, nodes)
                    if not math.isclose(pb, 0.0, abs_tol=0.000001):
                        n_prefix = prefix + (s, )
                        n_pb, n_pnb, nodes = next_hyps[n_prefix]
                        n_pnb = n_pnb + pb * ps
                        nodes = cur_nodes.copy()
                        nodes.append(dict(token=s, frame=t, prob=ps))
                        next_hyps[n_prefix] = (n_pb, n_pnb, nodes)
                else:
                    n_prefix = prefix + (s, )
                    n_pb, n_pnb, nodes = next_hyps[n_prefix]
                    if nodes:
                        if ps > nodes[-1]['prob']:
                            nodes.pop()
                            nodes.append(dict(token=s, frame=t, prob=ps))
                    else:
                        nodes = cur_nodes.copy()
                        nodes.append(dict(token=s, frame=t, prob=ps))
                    n_pnb = n_pnb + pb * ps + pnb * ps
                    next_hyps[n_prefix] = (n_pb, n_pnb, nodes)
        next_hyps = sorted(next_hyps.items(), key=lambda x: (x[1][0] + x[1][1]), reverse=True)
        cur_hyps = next_hyps[:path_beam_size]
    return cur_hyps


def hyps_of(cur_hyps):
    """loss.py:311: [(prefix, pb + pnb, nodes)]."""
    return [(y[0], y[1][0] + y[1][1], y[1][2]) for y in cur_hyps]


def is_sublist(main_list, check_list):
    """wekws/bin/score_ctc.py:88-103, verbatim behaviour (the last offset is never tried for a longer main list)."""
    if len(main_list) < len(check_list):
        return -1
    if len(main_list) == len(check_list):
        return 0 if tuple(main_list) == tuple(check_list) else -1
    for i in range(len(main_list) - len(check_list)):
        if main_list[i] == check_list[0]:
            for j in range(len(check_list)):
                if main_list[i + j] != check_list[j]:
                    break
            else:
                return i
    return -1


def ctc_keyword_hit(hyps, keywords_token):
    """wekws/bin/score_ctc.py:201-220 -> (word or None, hit_score, start, end)."""
    import math
    hit_keyword, hit_score, start, end = None, 1.0, 0, 0
    for one_hyp in hyps:
        prefix_ids, prefix_nodes = one_hyp[0], one_hyp[2]
        for word in keywords_token.keys():
            lab = keywords_token[word]['token_id']
            offset = is_sublist(prefix_ids, lab)
            if offset != -1:
                hit_keyword = word
                start = prefix_nodes[offset]['frame']
                end = prefix_nodes[offset + len(lab) - 1]['frame']
                for idx in range(offset, offset + len(lab)):
                    hit_score *= prefix_nodes[idx]['prob']
                break
        if hit_keyword is not None:
            hit_score = math.sqrt(hit_score)
            break
    return hit_keyword, hit_score, start, end
