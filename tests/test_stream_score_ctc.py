"""GPU tests of wekws_b200.stream_score_ctc (ctc_stream_score_kernel): the reference's score file and detections
(tests/golden/stream_score.npz) bit for bit, random peaky test sets against the oracle restatement
(oracle/kws_stream_score_oracle.py), batch-size and order invariance, the capacity relaunch, and FSMN-CTC / DS-TCN-CTC
posteriors end to end."""
import io

import numpy as np
import pytest
import torch

from oracle.kws_stream_score_oracle import ACTIVATED, stream_score
from tests.conftest import golden
from tests.test_spotter_host import golden_keywords
from tests.test_stream_score_host import golden_config, golden_records, golden_utterances
from tests.test_stream_spotter import _emitted_tokens, _model
from wekws_b200 import Fbank, _native, context_expansion, stream_score_ctc, synth, write_stream_ctc_scores
from wekws_b200.ctc import STREAM_SCORE_CAPACITY

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def padded(utts, pad_rows=3, seed=0):
    """[(key, probs (n, V))] -> (B, max n + pad_rows, V) CUDA tensor with random padding rows, lengths (B,)."""
    V = utts[0][1].shape[1]
    T = max(p.shape[0] for _, p in utts) + pad_rows
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(len(utts), T, V, generator=g).softmax(-1)
    for b, (_, p) in enumerate(utts):
        x[b, :p.shape[0]] = p
    return x.to(DEV), torch.tensor([p.shape[0] for _, p in utts], dtype=torch.int32)


def oracle(utts, kws, **cfg):
    return [[(w, s, st, en, fr) for w, s, st, en, fr in stream_score(p, kws, **cfg)[0]] for _, p in utts]


def test_golden_score_file_and_detections():
    """The reference's probabilities: the score-file text is identical, every activation (score as a double, keyword,
    start, end) equals the reference's log record, firing frames equal the oracle's."""
    g = golden("stream_score")
    kws = golden_keywords(g)
    words = list(kws)
    for c in range(int(g["nconfigs"])):
        cfg = golden_config(g, c)
        utts = golden_utterances(g, c)
        probs, lens = padded(utts, seed=c)
        res = stream_score_ctc(probs, lens, kws, **cfg)
        out = io.StringIO()
        write_stream_ctc_scores(out, [k for k, _ in utts], res)
        assert out.getvalue() == str(g[f"score_text{c}"])
        assert (res.overflow.cpu() == 0).all()
        got = [(k, words.index(w), s, st, en) for (k, _), dets in zip(utts, res.to_python())
               for w, s, st, en, _ in dets]
        want = [(k, kw, s, st, en) for k, kind, kw, s, st, en in golden_records(g, c) if kind == ACTIVATED]
        assert got == want
        assert res.to_python() == oracle(utts, kws, **cfg)


# keywords per vocabulary: a repeated token, tokens shared between keywords, ids near V
KEYWORDS = {48: {"k1": [5, 9, 17, 23], "k2": [31, 7, 23, 23], "k3": [9, 17]},
            2599: {"k1": [105, 2009, 17, 1023], "k2": [2598, 7, 1023, 1023], "k3": [2009, 17]}}


def random_test_set(B, V, max_len, seed, pad_rows=5):
    """Peaky posteriors built on the device: per utterance segments that spell keywords strongly, weakly (under a
    stronger blank), one frame per token or with long gaps, frames owned by a token outside the keywords (filtered
    out) and silence.  Lengths 0..max_len; every row past a length is random."""
    rng = np.random.RandomState(seed)
    kws = KEYWORDS[V]
    seqs = list(kws.values())
    other = 40 if V == 48 else 1500
    lens = rng.randint(0, max_len + 1, size=B)
    lens[rng.rand(B) < 0.05] = 0
    T = int(lens.max()) + pad_rows
    dom = np.full((B, T), -1, dtype=np.int64)
    strength = np.zeros((B, T), dtype=np.float32)
    weak = np.zeros((B, T), dtype=bool)
    for b in range(B):
        t = 0
        while t < lens[b]:
            kind = rng.randint(7)
            seq = seqs[rng.randint(len(seqs))]
            rows = []
            if kind == 0 or kind == 1:
                for tok in seq:
                    rows += [(tok, 9.0, False)] * int(rng.randint(1, 4)) + [(0, 9.0, False)] * int(rng.randint(0, 3))
            elif kind == 2:
                for tok in seq:
                    rows += [(tok, 6.3, True)] * 2 + [(0, 9.0, False)]
            elif kind == 3:
                for tok in seq:
                    rows += [(tok, 9.0, False)] * 2 + [(0, 9.0, False)] * int(rng.randint(5, 40))
            elif kind == 4:
                rows = [(other, 9.0, False)] * int(rng.randint(1, 10))
            else:
                rows = [(0, 9.0, False)] * int(rng.randint(1, 30))
            for tok, s, w in rows:
                if t >= T:
                    break
                dom[b, t], strength[b, t], weak[b, t] = tok, s, w
                t += 1
    gen = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(B, T, V, generator=gen, device=DEV) * 0.5
    d = torch.from_numpy(dom).to(DEV)
    s = torch.from_numpy(strength).to(DEV)
    has = d >= 0
    x.scatter_add_(2, d.clamp(min=0).unsqueeze(-1), (s * has).unsqueeze(-1))
    x[..., 0] += torch.from_numpy(weak).to(DEV) * 7.0                 # the stronger blank of the weak spelling
    return x.softmax(-1), torch.from_numpy(lens.astype(np.int32)), kws


CASES = [  # V, B, frame_skip, score_beam, path_beam
    (48, 1, 1, 3, 20), (48, 37, 3, 2, 3), (48, 300, 1, 3, 20), (48, 37, 1, 1, 1),
    (2599, 1, 3, 3, 20), (2599, 37, 1, 2, 20), (2599, 300, 3, 3, 3), (2599, 37, 3, 1, 1),
]
_activations = {}


@pytest.mark.parametrize("V,B,skip,sb,pb", CASES)
def test_random_matches_oracle(V, B, skip, sb, pb):
    probs, lens, kws = random_test_set(B, V, 1000, seed=V + B + 10 * skip + sb + pb)
    cfg = dict(score_beam_size=sb, path_beam_size=pb, threshold=0.3 if skip == 3 else 0.0, min_frames=5,
               max_frames=120 if B == 37 else 250, frame_skip=skip)
    res = stream_score_ctc(probs, lens, kws, **cfg)
    got = res.to_python()
    # a long stretch without activation can grow a prefix past MAX_PREFIX tokens: flagged, and not compared
    ok = (res.overflow.cpu() == 0).tolist()
    assert sum(ok) >= B - B // 10, ok
    for b in range(B):
        if ok[b]:
            want = stream_score(probs[b, :int(lens[b])].cpu(), kws, **cfg)[0]
            assert got[b] == want, (b, got[b], want)
    _activations[(V, B, skip, sb, pb)] = sum(len(d) for d, o in zip(got, ok) if o)


def test_random_activations_not_vacuous():
    if len(_activations) < len(CASES):
        pytest.skip("runs after the random tests")
    assert sum(_activations.values()) >= 500 and sum(v > 0 for v in _activations.values()) >= 6, _activations


def test_large_batch_equals_smaller_batches_in_any_order():
    B = 4096
    probs, lens, kws = random_test_set(B, 48, 300, seed=4096)
    cfg = dict(score_beam_size=3, path_beam_size=20, threshold=0.0, min_frames=5, max_frames=120, frame_skip=3)
    full = stream_score_ctc(probs, lens, kws, **cfg)
    whole = full.to_python()
    assert sum(len(d) for d in whole) >= 1000
    perm = torch.from_numpy(np.random.RandomState(1).permutation(B))
    parts = [None] * B
    for lo in range(0, B, 600):
        idx = perm[lo:lo + 600]
        sub = stream_score_ctc(probs[idx.to(DEV)], lens[idx], kws, **cfg).to_python()
        for j, b in enumerate(idx.tolist()):
            parts[b] = sub[j]
    assert parts == whole
    assert torch.equal(full.count.cpu(), torch.tensor([len(d) for d in whole], dtype=torch.int32))


def test_capacity_relaunch_keeps_every_activation():
    """An utterance that fires more often than the first launch has room for: every activation comes back, with
    exactly one more launch.  Otherwise a call is one launch."""
    V, kws = 48, {"k1": KEYWORDS[48]["k1"]}
    rows = []
    for _ in range(STREAM_SCORE_CAPACITY + 8):
        for tok in kws["k1"][:-1]:
            rows += [tok] * 2 + [0]
        rows += [kws["k1"][-1]] + [0] * 4
    x = torch.randn(3, len(rows), V) * 0.3
    x[0, torch.arange(len(rows)), torch.tensor(rows)] += 9.0
    x[1, :, 0] += 9.0
    x[2, :40, 40] += 9.0
    probs = x.softmax(-1).to(DEV)
    lens = torch.tensor([len(rows), len(rows), 40], dtype=torch.int32)
    torch.cuda.synchronize()
    n0 = _native.launch_count()
    res = stream_score_ctc(probs, lens, kws)
    got = res.to_python()
    assert _native.launch_count() - n0 == 2 and res.launches == 2
    assert len(got[0]) > STREAM_SCORE_CAPACITY and got[1] == [] and got[2] == []
    assert got == [stream_score(probs[b, :int(lens[b])].cpu(), kws)[0] for b in range(3)]
    n0 = _native.launch_count()
    res = stream_score_ctc(probs[1:], lens[1:], kws)
    assert _native.launch_count() - n0 == 1 and res.launches == 1


@pytest.mark.parametrize("name", ["fsmn", "ds_tcn"])
def test_end_to_end_matches_oracle(name):
    """FSMN-CTC (context 2/2, frame skip 3) and DS-TCN-CTC forward_softmax on padded features of different lengths,
    then stream_score_ctc, against the oracle decoding the same device posteriors."""
    ctx, skip, mel = ((2, 2), 3, 80) if name == "fsmn" else (None, 1, 40)
    fb = Fbank(mel)
    model = _model(name, mel * (5 if ctx else 1), 24, seed=5, scale=12.0)
    a, b, c = _emitted_tokens(model, fb, ctx, skip)
    kws = {"k_ab": [a, b], "k_bc": [b, c], "k_ca": [c, a]}
    B = 48
    # FSMN: at most 62 rows, so no prefix can outgrow MAX_PREFIX tokens whatever the random model emits
    feats = fb(synth.pcm_int16(B, 30400 if ctx else 16000 * 6, seed=21).to(DEV))
    lens = torch.from_numpy(np.random.RandomState(3).randint(0, feats.shape[1] + 1, size=B)).to(torch.int32)
    lens[:4] = torch.tensor([feats.shape[1], 0, 1, 7], dtype=torch.int32)
    if ctx:
        feats, lens = context_expansion(feats, ctx[0], ctx[1], skip, lens)
    probs, _ = model.forward_softmax(feats.contiguous())
    res = stream_score_ctc(probs, lens, kws, frame_skip=skip, max_frames=100)
    got = res.to_python()
    assert (res.overflow.cpu() == 0).all()
    for s in range(B):
        assert got[s] == stream_score(probs[s, :int(lens[s])].cpu(), kws, frame_skip=skip, max_frames=100)[0], s
    _e2e_activations[name] = sum(len(d) for d in got)


_e2e_activations = {}


def test_end_to_end_activations_not_vacuous():
    if len(_e2e_activations) < 2:
        pytest.skip("runs after the end-to-end tests")
    assert sum(_e2e_activations.values()) >= 5, _e2e_activations


def test_prefix_overflow_is_flagged():
    """Keyword tokens that never spell a keyword: a prefix of 64 tokens decodes as the reference does, one of 65 is
    flagged."""
    kws = {"k1": KEYWORDS[48]["k1"]}
    rows = [tok for i in range(65) for tok in ([5, 23][i % 2], 0)]
    x = torch.randn(2, len(rows), 48) * 0.3
    x[:, torch.arange(len(rows)), torch.tensor(rows)] += 9.0
    probs = x.softmax(-1).to(DEV)
    lens = torch.tensor([2 * 64, 2 * 65], dtype=torch.int32)
    res = stream_score_ctc(probs, lens, kws)
    assert res.overflow.cpu().tolist() == [0, 1]
    assert res.to_python()[0] == stream_score(probs[0, :128].cpu(), kws)[0] == []


def test_refuses_bad_input_on_device():
    probs = torch.full((2, 10, 8), 1 / 8, device=DEV)
    with pytest.raises(ValueError, match="lengths"):
        stream_score_ctc(probs, torch.tensor([10, 11], device=DEV), {"a": [1, 2]})
    with pytest.raises(ValueError, match="outside"):
        stream_score_ctc(probs, [10, 10], {"a": [1, 8]})
    res = stream_score_ctc(probs[:0], [], {"a": [1, 2]})
    assert res.to_python() == []
    res = stream_score_ctc(probs, [0, 0], {"a": [1, 2]})
    assert res.to_python() == [[], []]
