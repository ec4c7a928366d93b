"""Host tests of the online alarm rule of wekws_b200.ThresholdSpotter / ThresholdDecoder: a restatement of
threshold_spot_kernel, chunk by chunk, against the oracle of compute_det.py (pinned to the reference's own tool by
tests/test_oracle_pinned.py), the event-slot bound, the binding of the new entry points, and the refusals that need
no device."""
import math
import os
import re

import numpy as np
import pytest
import torch

from oracle import kws_oracle as O
from tests.conftest import REFERENCE, ROOT, golden, have_reference
from wekws_b200 import Fbank, Mfcc, ThresholdDecoder, ThresholdSpotter, init_model, model_config
from wekws_b200.spotter import event_slots, front_end_settings, trained_front_end


def round6(p):
    """The kernel's text_round6: the double Python parses back from '{:.6f}'.format(p)."""
    return np.rint(np.asarray(p, dtype=np.float32).astype(np.float64) * 1e6) / 1e6


class OnlineRule:
    """threshold_spot_kernel for one (stream, keyword), restated: the record (seen, next) and one scan per chunk."""

    def __init__(self, threshold: float, window_shift: int):
        self.th, self.ws = threshold, window_shift
        self.seen, self.next = 0, 0

    def __call__(self, probs):
        """probs: this chunk's posteriors; returns the frames (since reset) that fired, in order."""
        r6 = round6(probs)
        n, fired = len(r6), []
        i = max(self.next - self.seen, 0)
        while i < n:
            if r6[i] >= self.th:
                t = self.seen + i
                fired.append(t)
                self.next = t + self.ws
                i += self.ws
            else:
                i += 1
        self.seen += n
        return fired


def random_chunks(rng, n: int, ws: int):
    """Chunk sizes that add up to n: empty and one-frame chunks, chunks around window_shift and longer ones."""
    sizes, left = [], n
    while left > 0:
        s = int(rng.choice([0, 1, 1, 2, max(ws - 1, 0), ws, ws + 1, rng.randint(0, 60), rng.randint(0, 200)]))
        s = min(s, left)
        sizes.append(s)
        left -= s
    sizes.insert(int(rng.randint(0, len(sizes) + 1)), 0)
    return sizes


def test_online_rule_in_any_chunking_counts_the_reference_triggers():
    """The golden posteriors in random chunkings, every (window_shift, step) setting, every threshold of the sweep:
    each utterance's firings equal the triggers of oracle det_stats (compute_det.py), and no chunk fires more often
    than the event slots ceil(frames / window_shift) hold."""
    g = golden("det_stats")
    post, lens = g["post"], g["lens"]
    B, T, K = post.shape
    rng = np.random.RandomState(5)
    for ws, step in g["settings"].tolist():
        ws = int(ws)
        thr, _, want = O.det_stats(torch.from_numpy(post), torch.from_numpy(lens), step, ws)
        for b in range(B):
            n = int(lens[b])
            for _ in range(2):
                sizes = random_chunks(rng, n, ws)
                assert sum(sizes) == n and 0 in sizes
                for k in range(K):
                    for i, th in enumerate(thr):
                        rule, pos, fired = OnlineRule(th, ws), 0, []
                        for s in sizes:
                            got = rule(post[b, pos:pos + s, k])
                            assert len(got) <= event_slots(s, ws)
                            fired += got
                            pos += s
                        assert len(fired) == want[b][k][i], (ws, step, b, k, th, sizes)


def test_event_slot_bound_is_tight():
    """Threshold 0 fires every window_shift frames: a chunk that starts free fills ceil(frames / window_shift)
    slots exactly, whatever the chunking before it."""
    for ws in (1, 2, 7, 50):
        for n in (0, 1, ws - 1, ws, ws + 1, 3 * ws, 3 * ws + 1, 311):
            rule = OnlineRule(0.0, ws)
            assert len(rule(np.zeros(n, np.float32))) == event_slots(n, ws) == math.ceil(n / ws)
    assert event_slots(0, 5) == 0


def test_rule_edges_on_the_host():
    rule = OnlineRule(0.5, 4)
    assert rule(np.array([0.1, 0.9], np.float32)) == [1]          # fired on the chunk's last frame
    assert rule(np.array([0.9, 0.9, 0.9], np.float32)) == []       # frames 2..4 are suppressed
    assert rule(np.array([0.9, 0.9], np.float32)) == [5]
    # 0.4999995 and 0.5000005 both print as 0.500000 (round half to even on the exact binary value)
    assert OnlineRule(0.5, 1)(np.array([0.4999995, 0.5000005, 0.4999994], np.float32)) == [
        t for t, x in enumerate([0.4999995, 0.5000005, 0.4999994]) if float('{:.6f}'.format(np.float32(x))) >= 0.5]


def test_threshold_event_binding_matches_header(native):
    hdr = open(os.path.join(ROOT, "include", "wekws_b200.h")).read()
    code = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\} wekws_threshold_event;", code).group(1)
    numpy_type = {"int64_t": "<i8", "int32_t": "<i4", "float": "<f4"}
    fields = [(f.strip(), numpy_type[t]) for t, names in re.findall(r"(\w+)\s+([\w\s,]+);", body)
              for f in names.split(",")]
    assert fields == list(native.THRESHOLD_EVENT_DTYPE)
    assert np.dtype(native.THRESHOLD_EVENT_DTYPE).itemsize == native.THRESHOLD_EVENT_BYTES == 16
    for name in ("wekws_threshold_spot", "wekws_threshold_spot_state_bytes"):
        assert name in native.SIGNATURES
    assert native.lib().wekws_threshold_spot_state_bytes() == 16        # (seen, next) as two int64
    assert native.ABI_VERSION == 19


def _model(name="ds_tcn", idim=40, odim=2, activation="sigmoid", head=None):
    cfg = model_config(name, input_dim=idim, output_dim=odim, activation=activation)
    if head:
        cfg["classifier"] = dict(type=head, dropout=0.1)
    return init_model(cfg).eval()


def test_threshold_spotter_refuses_bad_arguments():
    m = _model()
    fb = Fbank(40)
    with pytest.raises(ValueError, match="per-frame"):
        ThresholdSpotter(_model("mdtc", 80, 2, head="global"), [0.5, 0.5], 2, frontend=Fbank(80))
    with pytest.raises(ValueError, match="per-frame"):
        ThresholdSpotter(_model("tcn", 40, 2, head="last"), [0.5, 0.5], 2, frontend=fb)
    with pytest.raises(ValueError, match="Sigmoid.*KeywordSpotter"):
        ThresholdSpotter(_model(activation="identity"), [0.5, 0.5], 2, frontend=fb)
    with pytest.raises(ValueError, match="one threshold per model output"):
        ThresholdSpotter(m, [0.5], 2, frontend=fb)
    with pytest.raises(ValueError, match="one threshold per model output"):
        ThresholdSpotter(m, [0.5, 0.5, 0.5], 2, frontend=fb)
    for bad in (float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError, match="finite"):
            ThresholdSpotter(m, [0.5, bad], 2, frontend=fb)
    for ws in (0, -3):
        with pytest.raises(ValueError, match="window_shift"):
            ThresholdSpotter(m, [0.5, 0.5], 2, frontend=fb, window_shift=ws)
    with pytest.raises(ValueError, match="keyword name"):
        ThresholdSpotter(m, [0.5, 0.5], 2, frontend=fb, keywords=["HI_XIAOWEN"])
    with pytest.raises(ValueError, match="left == right"):
        ThresholdSpotter(m, [0.5, 0.5], 2, frontend=fb, context=(2, 1))
    with pytest.raises(ValueError, match="inputs per frame"):
        ThresholdSpotter(m, [0.5, 0.5], 2, frontend=Fbank(80))
    with pytest.raises(RuntimeError, match="ThresholdSpotter runs on CUDA only"):     # no CPU fallback
        ThresholdSpotter(m, [0.5, 0.5], 2, frontend=fb)
    with pytest.raises(ValueError, match="finite"):
        ThresholdDecoder(2, [0.5, float("nan")], 50)
    with pytest.raises(ValueError, match="window_shift"):
        ThresholdDecoder(2, [0.5], 0)
    with pytest.raises(ValueError, match="at least one threshold"):
        ThresholdDecoder(2, [], 50)


def test_from_config_reads_the_recipe_front_end():
    """hi_xiaowen ds_tcn.yaml's dataset_conf: 40 mel bins, 25 / 10 ms, no context, no frame skip."""
    conf = {"dataset_conf": {"fbank_conf": {"num_mel_bins": 40, "frame_shift": 10, "frame_length": 25, "dither": 0.1},
                             "feature_extraction_conf": {"num_mel_bins": 40, "frame_shift": 10, "frame_length": 25}}}
    fb, context, skip, shift = front_end_settings(conf)
    assert fb.feature_dim == 40 and (fb.win, fb.shift) == (400, 160) and context is None and skip == 1
    assert shift == 0.01
    with pytest.raises(RuntimeError, match="CUDA"):
        ThresholdSpotter.from_config(conf, _model(), 2, thresholds=[0.5, 0.5])


# the feature sections of the max-pooling recipes' dataset_conf (examples/*/s0/conf/*.yaml)
_MFCC_80 = {"feature_extraction_conf": {"feature_type": "mfcc", "num_ceps": 80, "num_mel_bins": 80, "frame_shift": 10,
                                        "frame_length": 25, "dither": 1.0}}
_FBANK_40 = {"feature_extraction_conf": {"feature_type": "fbank", "num_mel_bins": 40, "frame_shift": 10,
                                         "frame_length": 25, "dither": 1.0}}
_FEATS_FBANK_40 = {"feats_type": "fbank", "fbank_conf": {"num_mel_bins": 40, "frame_shift": 10, "frame_length": 25,
                                                         "dither": 0.1}}
RECIPE_FEATURES = {"hi_xiaowen/mdtc": _MFCC_80, "hi_xiaowen/mdtc_small": _MFCC_80, "hi_xiaowen/ds_tcn": _FEATS_FBANK_40,
                   "hi_xiaowen/tcn": _FBANK_40, "hi_xiaowen/gru": _FBANK_40, "hey_snips/ds_tcn": _FEATS_FBANK_40,
                   "hey_snips/mdtc_small": _MFCC_80}


def _check_front_end(recipe, ds):
    fe, context, skip = trained_front_end({"dataset_conf": ds})
    assert context is None and skip == 1 and (fe.win, fe.shift) == (400, 160)
    if recipe.endswith("mdtc") or recipe.endswith("mdtc_small"):
        assert isinstance(fe, Mfcc) and fe.num_ceps == 80 and fe.num_mel_bins == 80 and fe.feature_dim == 80
        assert fe.lifter is not None                       # kaldi.mfcc's default cepstral_lifter 22
    else:
        assert type(fe) is Fbank and fe.feature_dim == 40


@pytest.mark.parametrize("recipe", list(RECIPE_FEATURES))
def test_from_config_builds_the_front_end_the_recipe_trains_on(recipe):
    """The mdtc / mdtc_small recipes train on MFCC (feature_type: mfcc, 80 cepstra of 80 mel bins): from_config
    streams Mfcc for them, Fbank for the others.  A CPU model gets as far as the CUDA refusal, so the widths agree."""
    ds = RECIPE_FEATURES[recipe]
    _check_front_end(recipe, ds)
    name = recipe.split("/")[1]
    mel = 80 if name.startswith("mdtc") else 40
    with pytest.raises(RuntimeError, match="CUDA"):
        ThresholdSpotter.from_config({"dataset_conf": ds}, _model(name, mel, 2), 2, thresholds=[0.5, 0.5])


@pytest.mark.skipif(not have_reference(), reason="the reference's recipe configs are not present")
@pytest.mark.parametrize("recipe", list(RECIPE_FEATURES))
def test_front_end_of_the_reference_recipe_files(recipe):
    """The same, read from the reference's own yaml files."""
    import yaml
    site, name = recipe.split("/")
    with open(os.path.join(REFERENCE, "examples", site, "s0", "conf", name + ".yaml")) as f:
        ds = yaml.safe_load(f)["dataset_conf"]
    _check_front_end(recipe, ds)


def test_trained_front_end_refuses_an_unknown_feature_type():
    with pytest.raises(ValueError, match="'spectrogram'"):
        trained_front_end({"dataset_conf": {"feature_extraction_conf": {
            "feature_type": "spectrogram", "num_mel_bins": 40, "frame_shift": 10, "frame_length": 25}}})
    fe, _, _ = trained_front_end({"dataset_conf": {"feats_type": "mfcc", "mfcc_conf": {
        "num_ceps": 40, "num_mel_bins": 80, "frame_shift": 10, "frame_length": 25}}})
    assert isinstance(fe, Mfcc) and fe.feature_dim == 40
