"""CPU tests of the streaming keyword spotter: the oracle restatement (oracle/kws_spotter_oracle.py) against the
reference's own KeyWordSpotter (tests/golden/spotter.npz, and live when the reference sources are present), the host
integer mirror that predicts every stream's frame count, and argument validation."""
import math

import numpy as np
import pytest
import torch

from oracle import kws_oracle as O
from oracle.kws_spotter_oracle import SpotterOracle
from tests.conftest import golden, have_reference
from wekws_b200 import KeywordSpotter, init_model, model_config
from wekws_b200.spotter import StreamMirror


def case_pcm(seed, n):
    return np.random.RandomState(seed + 1000).randint(-3000, 3001, size=n).astype(np.int16)


def golden_case(g, i):
    c = dict(mel=int(g[f"mel{i}"]), skip=int(g[f"skip{i}"]), threshold=float(g[f"threshold{i}"]),
             min_frames=int(g[f"min_frames{i}"]), max_frames=int(g[f"max_frames{i}"]),
             interval_frames=int(g[f"interval_frames{i}"]))
    ctx = tuple(int(x) for x in g[f"context{i}"])
    c["context"] = None if ctx == (0, 0) else ctx
    return c


def golden_keywords(g):
    off = g["kw_offsets"]
    return {str(w): [int(t) for t in g["kw_tokens"][off[k]:off[k + 1]]] for k, w in enumerate(g["kw_names"])}


def decode_result(row, words):
    state = int(row[0])
    if state == -1:
        return {}
    if state == 0:
        return {"state": 0, "keyword": None, "start": None, "end": None, "score": None}
    return {"state": 1, "keyword": words[int(row[1])], "start": float(row[2]), "end": float(row[3]),
            "score": float(row[4])}


class ScriptedProbs:
    """Model step that hands out the next T rows of fixed probabilities."""

    def __init__(self, probs):
        self.probs, self.pos = torch.as_tensor(probs), 0

    def __call__(self, feats):
        T = feats.shape[0]
        out = self.probs[self.pos:self.pos + T]
        assert out.shape[0] == T
        self.pos += T
        return out

    def reset(self):
        pass


def hyps_equal(got, g, i):
    """Oracle cur_hyps == the reference's final cur_hyps stored in the golden (pb, pnb, nodes exact)."""
    n = len(g[f"hyp_len{i}"])
    assert len(got) == n
    for j, (prefix, (pb, pnb, nodes)) in enumerate(got):
        L = int(g[f"hyp_len{i}"][j])
        assert list(prefix) == g[f"hyp_tok{i}"][j, :L].tolist()
        assert [nd["frame"] for nd in nodes] == g[f"hyp_frame{i}"][j, :L].tolist()
        assert [nd["prob"] for nd in nodes] == g[f"hyp_prob{i}"][j, :L].tolist()
        assert pb == float(g[f"hyp_pb{i}"][j]) and pnb == float(g[f"hyp_pnb{i}"][j])


def test_oracle_matches_reference_golden():
    g = golden("spotter")
    kws = golden_keywords(g)
    words = list(kws)
    for i in range(int(g["ncases"])):
        c = golden_case(g, i)
        lens = g[f"lens{i}"]
        pcm = case_pcm(int(g[f"seed{i}"]), int(lens.sum()))
        assert int(pcm.astype(np.int64).sum()) == int(g[f"pcm_sum{i}"])
        o = SpotterOracle(kws, ScriptedProbs(g[f"probs{i}"]), num_mel_bins=c["mel"], context=c["context"],
                          frame_skip=c["skip"], threshold=c["threshold"], min_frames=c["min_frames"],
                          max_frames=c["max_frames"], interval_frames=c["interval_frames"])
        feats_ref, fpos, pos = g[f"feats{i}"], 0, 0
        plain = o.accept_wave
        seen = []
        o.accept_wave = lambda s: seen.append(plain(s)) or seen[-1]
        for k, n in enumerate(lens):
            got = o.forward(pcm[pos:pos + n])
            pos += n
            want = decode_result(g[f"result{i}"][k], words)
            assert got.keys() == want.keys(), (i, k, got, want)
            for key in got:                    # scores as doubles, start / end as the products Python formed
                assert got[key] == want[key] or (want[key] != want[key] and got[key] is None), (i, k, key, got, want)
            f = seen[-1]
            assert (-1 if f is None else f.shape[0]) == int(g[f"frames{i}"][k])
            assert len(o.wave_remained) == int(g[f"rem{i}"][k])
            if f is not None and k < int(g["feat_chunks"]):
                ref = feats_ref[fpos:fpos + f.shape[0]]
                fpos += f.shape[0]
                assert float(np.abs(f.numpy() - ref).max()) <= 1e-3, (i, k)
        assert o.model_step.pos == len(g[f"probs{i}"])
        hyps_equal(o.cur_hyps, g, i)


def test_mirror_matches_reference_golden():
    """Frame count and PCM remainder after every golden chunk, from the chunk lengths alone."""
    g = golden("spotter")
    for i in range(int(g["ncases"])):
        c = golden_case(g, i)
        L = c["context"][0] if c["context"] else 0
        m = StreamMirror(1, 400, 160, L, L, c["skip"])
        for k, n in enumerate(g[f"lens{i}"]):
            plan = m.advance([n])
            frames = int(g[f"frames{i}"][k])
            assert int(plan["nout"][0]) == max(frames, 0), (i, k)
            assert (plan["nfeat"][0] == 0) == (frames == -1)
            assert int(m.rem_len[0]) == int(g[f"rem{i}"][k]), (i, k)


def _reference():
    from oracle.make_spotter_golden import import_reference
    return import_reference()


def _random_lengths(rng, n, min_len):
    pick = [lambda: 4800, lambda: int(rng.randint(min_len, 900)), lambda: int(rng.randint(min_len, 6000)),
            lambda: int(rng.randint(min_len, 2000))]
    if min_len == 0:
        pick.append(lambda: 0)
    return [pick[int(rng.randint(len(pick)))]() for _ in range(n)]


@pytest.mark.skipif(not have_reference(), reason="reference sources not present")
def test_mirror_matches_reference_live():
    """1000 random chunk-length sequences through the reference's accept_wave: same frame count (None = held) and
    PCM remainder after every chunk.  Without context expansion the reference raises below one window, so those
    sequences keep every chunk >= 400 samples."""
    from oracle.make_spotter_golden import ScriptedModel, reference_spotter
    S = _reference()
    rng = np.random.RandomState(5)
    pcm = rng.randint(-3000, 3001, size=6000).astype(np.int16)
    for seq in range(1000):
        context, skip = [((2, 2), 3), (None, 1), (None, 3), ((2, 2), 1)][seq % 4]
        lens = _random_lengths(rng, 6, 0 if context else 400)
        k = reference_spotter(S, ScriptedModel(None), 40, context, skip)
        m = StreamMirror(1, 400, 160, *(context or (0, 0)), skip)
        for n in lens:
            f = k.accept_wave(pcm[:n].tobytes())
            plan = m.advance([n])
            assert int(plan["nout"][0]) == (0 if f is None else f.size(0)), (seq, lens)
            assert int(m.rem_len[0]) == len(k.wave_remained), (seq, lens)


@pytest.mark.skipif(not have_reference(), reason="reference sources not present")
def test_oracle_matches_reference_live():
    """The restatement against the reference's own KeyWordSpotter on further random chunk sequences and detection
    settings: every return value (scores as doubles) and the final hypotheses."""
    from oracle.make_spotter_golden import KEYWORDS, ScriptedModel, reference_spotter, scripted_logits
    S = _reference()
    rng = np.random.RandomState(9)
    for seq in range(6):
        context, skip, mel = [((2, 2), 3, 80), (None, 1, 40), ((1, 1), 2, 40)][seq % 3]
        params = dict(threshold=float(rng.choice([0.0, 0.5])), min_frames=int(rng.choice([5, 10])),
                      max_frames=int(rng.choice([80, 250])), interval_frames=int(rng.choice([20, 50, 100])))
        logits = scripted_logits(2000, 100 + seq, skip, params["max_frames"])
        k = reference_spotter(S, ScriptedModel(logits), mel, context, skip, **params)
        o = SpotterOracle(KEYWORDS, ScriptedProbs(logits.softmax(1)), num_mel_bins=mel, context=context,
                          frame_skip=skip, **params)
        lens = _random_lengths(rng, 30, 0 if context and context[1] == 2 else 600)
        pcm = rng.randint(-3000, 3001, size=sum(lens)).astype(np.int16)
        pos = 0
        for n in lens:
            want = k.forward(pcm[pos:pos + n].tobytes())
            got = o.forward(pcm[pos:pos + n])
            pos += n
            assert got == want, (seq, got, want)
        assert [(h[0], h[1][0], h[1][1], [(d["token"], d["frame"], d["prob"]) for d in h[1][2]]) for h in o.cur_hyps] \
            == [(h[0], h[1][0], h[1][1], [(d["token"], d["frame"], d["prob"]) for d in h[1][2]]) for h in k.cur_hyps]


def test_oracle_holds_short_buffers_without_context():
    """The one deliberate difference: without context expansion a buffer shorter than one window is held (the
    reference raises and loses it) and the call returns {}."""
    probs = torch.full((100, 8), 1 / 8)
    o = SpotterOracle({"a": [1, 2]}, ScriptedProbs(probs), num_mel_bins=40)
    assert o.forward(np.zeros(300, np.int16)) == {} and len(o.wave_remained) == 300
    assert o.forward(np.zeros(99, np.int16)) == {} and len(o.wave_remained) == 399
    r = o.forward(np.zeros(1, np.int16))
    assert r["state"] == 0 and len(o.wave_remained) == 240
    m = StreamMirror(1, 400, 160, 0, 0, 1)
    assert [int(m.advance([n])["nout"][0]) for n in (300, 99, 1)] == [0, 0, 1] and int(m.rem_len[0]) == 240


def test_spotter_refuses_bad_arguments():
    fsmn = init_model(model_config("fsmn", input_dim=400, output_dim=48)).eval()
    kws = {"a": [5, 9]}
    from wekws_b200 import Fbank
    with pytest.raises(ValueError, match="left == right"):
        KeywordSpotter(fsmn, kws, 2, frontend=Fbank(80), context=(2, 1), frame_skip=3)
    with pytest.raises(ValueError, match="left == right"):
        StreamMirror(2, 400, 160, 3, 2, 1)
    with pytest.raises(ValueError, match="path_beam_size"):
        KeywordSpotter(fsmn, kws, 2, frontend=Fbank(80), context=(2, 2), path_beam_size=21)
    with pytest.raises(ValueError, match="score_beam_size"):
        KeywordSpotter(fsmn, kws, 2, frontend=Fbank(80), context=(2, 2), score_beam_size=4)
    with pytest.raises(ValueError, match="keyword"):
        KeywordSpotter(fsmn, {"long": list(range(1, 66))}, 2, frontend=Fbank(80), context=(2, 2))
    with pytest.raises(ValueError, match="outside"):
        KeywordSpotter(fsmn, {"a": [5, 48]}, 2, frontend=Fbank(80), context=(2, 2))
    with pytest.raises(ValueError, match="inputs per frame"):
        KeywordSpotter(fsmn, kws, 2, frontend=Fbank(80), context=None)
    cfg = model_config("mdtc", output_dim=11)
    cfg["classifier"] = dict(type="global", dropout=0.1)
    head = init_model(cfg).eval()
    with pytest.raises(ValueError, match="per-frame"):
        KeywordSpotter(head, {"a": [1]}, 2, frontend=Fbank(80))
    with pytest.raises(RuntimeError, match="CUDA"):                       # a CPU model: no CPU fallback
        KeywordSpotter(fsmn, kws, 2, frontend=Fbank(80), context=(2, 2))
