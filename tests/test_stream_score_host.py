"""CPU tests of streaming CTC scoring and the CTC DET statistics: the oracle restatement
(oracle/kws_stream_score_oracle.py) against the reference's own stream_score_ctc.py main() (tests/golden/stream_score.npz,
and live when the reference sources are present), ctc_det_stats / write_ctc_det_stats against compute_det_ctc.py
(tests/golden/det_ctc.npz, and live), and argument validation."""
import io
import math
import os

import numpy as np
import pytest
import torch

from oracle.kws_stream_score_oracle import ACTIVATED, BAD_DURATION, score_lines, stream_score
from tests.conftest import golden, have_reference
from wekws_b200 import ctc_det_stats, space_mixed_label, stream_score_ctc, write_ctc_det_stats


def golden_keywords(g):
    off = g["kw_offsets"]
    return {str(w): [int(t) for t in g["kw_tokens"][off[k]:off[k + 1]]] for k, w in enumerate(g["kw_names"])}


def golden_config(g, c):
    return dict(score_beam_size=int(g[f"score_beam{c}"]), path_beam_size=int(g[f"path_beam{c}"]),
                threshold=float(g[f"threshold{c}"]), min_frames=int(g[f"min_frames{c}"]),
                max_frames=int(g[f"max_frames{c}"]), frame_skip=int(g[f"frame_skip{c}"]))


def golden_utterances(g, c):
    """[(key, probs (n, V))] in score-file order."""
    rows = torch.from_numpy(g[f"probs{c}"])
    out, pos = [], 0
    for key, n in zip(g[f"keys{c}"], g[f"lengths{c}"]):
        out.append((str(key), rows[pos:pos + int(n)]))
        pos += int(n)
    assert pos == rows.shape[0]
    return out


def golden_records(g, c):
    """[(key, kind, keyword index, score, start, end)] of the reference's detect log lines."""
    return [(str(k), int(r[0]), int(r[1]), float(s), int(r[2]), int(r[3]))
            for k, r, s in zip(g[f"rec_key{c}"], g[f"rec{c}"].reshape(-1, 4), g[f"rec_score{c}"])]


def oracle_run(utts, kws, cfg):
    """Score-file text and [(key, kind, keyword index, score, start, end)] of the restatement."""
    words = list(kws)
    text, records = [], []
    for key, p in utts:
        dets, events = stream_score(p, kws, **cfg)
        text += score_lines(key, dets)
        records += [(key, kind, words.index(w), s, st, en) for kind, w, s, st, en, _ in events]
    return "".join(text), records


def records_equal(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a[:3] == b[:3] and a[4:] == b[4:], (a, b)
        if a[1] != BAD_DURATION:                 # the duration log line does not print the score
            assert a[3] == b[3], (a, b)          # doubles, bitwise: repr round-trips


def test_oracle_matches_reference_golden():
    g = golden("stream_score")
    kws = golden_keywords(g)
    for c in range(int(g["nconfigs"])):
        cfg = golden_config(g, c)
        text, records = oracle_run(golden_utterances(g, c), kws, cfg)
        assert text == str(g[f"score_text{c}"])
        records_equal(records, golden_records(g, c))


def test_golden_covers_the_quirks():
    """The fixture exercises repeated activations, stale hits square-rooted towards 1 and a late activation."""
    g = golden("stream_score")
    acts, late = {}, 0
    for c in range(int(g["nconfigs"])):
        recs = golden_records(g, c)
        for i, r in enumerate(recs):
            if r[1] == ACTIVATED:
                acts[r[0]] = acts.get(r[0], 0) + 1
                p = recs[i - 1]
                late += i > 0 and p[0] == r[0] and p[1] != ACTIVATED and p[2] == r[2] and p[4:] == r[4:]
    assert max(acts.values()) >= 2 and late >= 1
    assert any(int(n) == 0 for c in range(int(g["nconfigs"])) for n in g[f"lengths{c}"])


@pytest.mark.skipif(not have_reference(), reason="reference sources not present")
@pytest.mark.parametrize("c", [0, 1])
def test_oracle_matches_reference_live(c):
    """About 200 random peaky utterances per configuration through the reference's main() and the restatement."""
    from oracle import make_stream_score_golden as M
    S = M.import_reference()
    cfg = M.CONFIGS[c]
    batches = M.make_batches([40, 50, 60, 50], 500 + c, hand=False)
    text, recs, decoded = M.run_reference(S, cfg, batches)
    utts = [(k, p[b, :int(n[b])]) for ks, p, n in decoded for b, k in enumerate(ks)]
    kws = M.keyword_tokens()
    words = list(kws)
    got_text, got = oracle_run(utts, kws, dict(score_beam_size=cfg["score_beam"], path_beam_size=cfg["path_beam"],
                                               threshold=cfg["threshold"], min_frames=cfg["min_frames"],
                                               max_frames=cfg["max_frames"], frame_skip=cfg["frame_skip"]))
    assert got_text == text
    want = [(k, kind, words.index(w), s, st, en) for k, kind, w, s, st, en in recs]
    records_equal(got, want)
    assert sum(r[1] == ACTIVATED for r in want) >= 20


def _det_case(g, i):
    kws = str(g[f"keywords{i}"])
    labels = [(str(k), str(t), float(d)) for k, t, d in zip(g[f"label_key{i}"], g[f"label_txt{i}"], g[f"label_dur{i}"])]
    return {k: "".join(k) for k in kws.split(",")}, str(g[f"score_text{i}"]), labels, float(g[f"step{i}"])


def test_ctc_det_stats_matches_reference_golden(tmp_path):
    g = golden("det_ctc")
    for i in range(int(g["ncases"])):
        kws, text, labels, step = _det_case(g, i)
        d = tmp_path / str(i)
        d.mkdir()
        paths = write_ctc_det_stats(str(d), ctc_det_stats(io.StringIO(text), labels, kws, step))
        want = dict(zip([str(n) for n in g[f"stats_names{i}"]], [str(t) for t in g[f"stats_text{i}"]]))
        assert sorted(os.path.basename(p) for p in paths) == sorted(want)
        for p in paths:
            with open(p, encoding="utf8") as f:
                assert f.read() == want[os.path.basename(p)], p


@pytest.mark.skipif(not have_reference(), reason="reference sources not present")
def test_ctc_det_stats_matches_reference_live(tmp_path):
    """Fresh random label files and score files of both formats through compute_det_ctc.py."""
    from oracle import make_det_ctc_golden as M
    g = golden("stream_score")
    score_text = "".join(str(g[f"score_text{c}"]) for c in range(int(g["nconfigs"])))
    keys = [str(k) for c in range(int(g["nconfigs"])) for k in g[f"keys{c}"]]
    for seed in range(4):
        rng = np.random.RandomState(100 + seed)
        off_text, off_labels = M.offline_case(rng)
        for kws, text, labels, step in [("abcd,efdd", score_text, M.stream_labels(keys, score_text, rng), 0.01),
                                        ("你好问问,hey", off_text, off_labels, [0.01, 0.02, 0.05, 0.1][seed])]:
            want = M.run_reference(text, labels, kws, step)
            d = tmp_path / f"{seed}_{len(kws)}"
            d.mkdir()
            paths = write_ctc_det_stats(str(d), ctc_det_stats(text, labels, M.true_keywords(kws), step))
            got = {}
            for p in paths:
                with open(p, encoding="utf8") as f:
                    got[os.path.basename(p)] = f.read()
            assert got == want


def test_space_mixed_label():
    assert space_mixed_label("你好 ABCD呀 hi!") == "你 好 abcd 呀 hi!"
    assert space_mixed_label("abab ab") == "abab ab"


def test_ctc_det_stats_refuses_bad_input():
    kws = {"abcd": "abcd"}
    lines = ["u1 detected abcd 0.900\n", "u2 rejected\n", "u3 detected abcd 0.300\n", "u3 rejected\n"]
    rows = ctc_det_stats(lines, [("u1", "abcd", 1.0), ("u2", "x", 3600.0), ("u3", "y", 3600.0)], kws, 0.5)["abcd"]
    assert rows == [(0.0, 0.5, 0.0), (0.5, 5e-7, 0.0), (1.0, 5e-7, 1.0)]
    with pytest.raises(ValueError, match="positive"):
        ctc_det_stats(lines, [("u2", "x", 1.0)], kws)
    with pytest.raises(ValueError, match="negative"):
        ctc_det_stats(lines, [("u1", "abcd", 1.0)], kws)
    with pytest.raises(ValueError, match="score file"):
        ctc_det_stats(lines, [("u4", "abcd", 1.0)], kws)


def test_stream_score_refuses_bad_arguments():
    probs = torch.full((2, 10, 8), 1 / 8)
    kws = {"a": [1, 2]}
    with pytest.raises(ValueError, match="score_beam_size"):
        stream_score_ctc(probs, [10, 10], kws, score_beam_size=4)
    with pytest.raises(ValueError, match="path_beam_size"):
        stream_score_ctc(probs, [10, 10], kws, path_beam_size=21)
    with pytest.raises(ValueError, match="frame_stride"):
        stream_score_ctc(probs, [10, 10], kws, frame_skip=0)
    with pytest.raises(ValueError, match="keyword"):
        stream_score_ctc(probs, [10, 10], {})
    with pytest.raises(ValueError, match="float32"):
        stream_score_ctc(probs.double(), [10, 10], kws)
    with pytest.raises(ValueError, match="float32"):
        stream_score_ctc(probs[0], [10], kws)
    with pytest.raises(ValueError, match="lengths"):
        stream_score_ctc(probs, [10, 11], kws)
    with pytest.raises(ValueError, match="lengths"):
        stream_score_ctc(probs, [10, -1], kws)
    with pytest.raises(ValueError, match="lengths"):
        stream_score_ctc(probs, [10], kws)
    with pytest.raises(ValueError, match="outside"):
        stream_score_ctc(probs, [10, 10], {"a": [1, 8]})
    with pytest.raises(RuntimeError, match="CUDA"):                       # no CPU fallback
        stream_score_ctc(probs, [10, 10], kws)
    assert math.isfinite(float(probs.sum()))
