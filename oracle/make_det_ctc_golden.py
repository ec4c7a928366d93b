#!/usr/bin/env python
"""Golden vectors for the CTC DET statistics (test infrastructure): runs the REFERENCE's wekws/bin/compute_det_ctc.py
as __main__ (runpy) with matplotlib, matplotlib.pyplot (no-op plotting), pypinyin and the wenet tokenizer stubbed, on
  1. the score files of tests/golden/stream_score.npz (both configurations, one file) and
  2. an offline-style score file (score_ctc.py's format: one line per utterance) with a CJK and a Latin keyword,
each with a synthetic label file that mixes Latin and CJK text, holds a duplicate key and positives detected as the
wrong keyword.  Stores the inputs and every stats.<keyword>.txt in tests/golden/det_ctc.npz.
      python oracle/make_det_ctc_golden.py"""
import glob
import json
import os
import runpy
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFERENCE = "/root/reference"


class CharTokenizer:
    def __init__(self, *args, **kwargs):
        pass

    def tokenize(self, line):
        strs = line.split(" ")
        return strs, [ord(s) for s in strs]


def _noop(*args, **kwargs):
    return None


def install_stubs():
    plt = types.ModuleType("matplotlib.pyplot")
    plt.rcParams = {}
    for name in ("figure", "plot", "xlim", "ylim", "xticks", "yticks", "xlabel", "ylabel", "grid", "legend", "savefig"):
        setattr(plt, name, _noop)
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = plt
    sys.modules["matplotlib"], sys.modules["matplotlib.pyplot"] = mpl, plt
    pin = types.ModuleType("pypinyin")
    pin.lazy_pinyin = lambda s: [s]
    sys.modules["pypinyin"] = pin
    for name in ("wenet", "wenet.text"):
        sys.modules.setdefault(name, types.ModuleType(name))
    tok = types.ModuleType("wenet.text.char_tokenizer")
    tok.CharTokenizer = CharTokenizer
    sys.modules["wenet.text.char_tokenizer"] = tok


def run_reference(score_text, labels, keywords, step):
    """compute_det_ctc.py on these inputs -> {stats file name: its text}.  labels: [(key, txt, duration)]."""
    install_stubs()
    with tempfile.TemporaryDirectory() as tmp:
        score = os.path.join(tmp, "score.txt")
        with open(score, "w", encoding="utf8") as f:
            f.write(score_text)
        data = os.path.join(tmp, "data.list")
        with open(data, "w", encoding="utf8") as f:
            for key, txt, dur in labels:
                f.write(json.dumps(dict(key=key, wav=f"{key}.wav", txt=txt, duration=dur), ensure_ascii=False) + "\n")
        stats = os.path.join(tmp, "stats")
        os.makedirs(stats)
        argv = sys.argv
        # --keywords goes through .encode('utf-8').decode('unicode_escape') (:212): pass non-ASCII as \u escapes
        sys.argv = ["compute_det_ctc.py", "--test_data", data, "--score_file", score, "--stats_dir", stats,
                    "--keywords", keywords.encode("unicode_escape").decode("ascii"), "--step", repr(step)]
        try:
            runpy.run_path(os.path.join(REFERENCE, "wekws", "bin", "compute_det_ctc.py"), run_name="__main__")
        finally:
            sys.argv = argv
        out = {}
        for p in sorted(glob.glob(os.path.join(stats, "stats.*.txt"))):
            with open(p, encoding="utf8") as f:
                out[os.path.basename(p)] = f.read()
    return out


def true_keywords(keywords):
    """compute_det_ctc.py:220-223 with the character tokenizer: {keyword: its token string}."""
    return {k: "".join(k) for k in keywords.split(",")}


POS = {"abcd": ["abcd", "你好 abcd 呀", "Hi ABCD there"], "efdd": ["efdd", "efdd 问问", "小 efdd"]}
NEG = ["你好问问", "hello world", "abcd!", "ab cd", "嗨 小 问", "efd d", "xabcd"]


def stream_labels(keys, score_text, rng):
    """Labels for the stream golden's utterances: positives of both keywords (some detected as the other one),
    negatives, mixed Latin / CJK, one duplicate key."""
    detected = {}
    for line in score_text.splitlines():
        arr = line.split()
        if arr[1] == "detected":
            detected.setdefault(arr[0], arr[2])
    labels = []
    for i, key in enumerate(keys):
        r = rng.rand()
        if key in detected and r < 0.6:
            kw = detected[key] if r < 0.45 else ("efdd" if detected[key] == "abcd" else "abcd")   # some wrong
            txt = POS[kw][int(rng.randint(len(POS[kw])))]
        elif r < 0.75:
            kw = ["abcd", "efdd"][int(rng.randint(2))]
            txt = POS[kw][int(rng.randint(len(POS[kw])))]
        else:
            txt = NEG[int(rng.randint(len(NEG)))]
        labels.append((key, txt, round(float(rng.uniform(0.5, 6.0)), 2)))
    labels.append((keys[3], NEG[0], 2.5))                 # duplicate key: entry replaced, duration added again
    return labels


def offline_case(rng):
    """An offline-style score file (score_ctc.py: first line per key) with keywords 你好问问 and hey."""
    keys = [f"off{i:03d}" for i in range(60)]
    lines, labels = [], []
    for key in keys:
        r = rng.rand()
        truth = "你好问问" if r < 0.35 else ("hey" if r < 0.6 else None)
        u = rng.rand()
        if u < 0.55:
            word = truth if (truth is not None and u < 0.45) else ["你好问问", "hey"][int(rng.randint(2))]
            lines.append(f"{key} detected {word} {rng.rand():.3f}\n")
        else:
            lines.append(f"{key} rejected\n")
        if rng.rand() < 0.1:                                # a second line for the key: the first one wins
            lines.append(f"{key} detected hey {rng.rand():.3f}\n")
        txt = {"你好问问": ["你好问问", "嗯 你好问问 hello", "你 好 问 问"], "hey": ["hey", "Hey 你好", "oh hey there"],
               None: ["你好", "heyy", "hello 问问", "they"]}[truth]
        labels.append((key, txt[int(rng.randint(len(txt)))], round(float(rng.uniform(0.5, 8.0)), 2)))
    labels.append((keys[7], "hey", 1.25))
    return "".join(lines), labels


def main():
    rng = np.random.RandomState(31)
    g = np.load(os.path.join(ROOT, "tests", "golden", "stream_score.npz"))
    score_text = "".join(str(g[f"score_text{c}"]) for c in range(int(g["nconfigs"])))
    keys = [str(k) for c in range(int(g["nconfigs"])) for k in g[f"keys{c}"]]
    cases = [("abcd,efdd", score_text, stream_labels(keys, score_text, rng), 0.01)]
    off_text, off_labels = offline_case(rng)
    cases.append(("你好问问,hey", off_text, off_labels, 0.05))
    out = {"ncases": np.array(len(cases))}
    for i, (kws, text, labels, step) in enumerate(cases):
        stats = run_reference(text, labels, kws, step)
        assert len(stats) == len(kws.split(",")), stats.keys()
        out[f"keywords{i}"] = np.array(kws)
        out[f"score_text{i}"] = np.array(text)
        out[f"label_key{i}"] = np.array([k for k, _, _ in labels])
        out[f"label_txt{i}"] = np.array([t for _, t, _ in labels])
        out[f"label_dur{i}"] = np.array([d for _, _, d in labels], dtype=np.float64)
        out[f"step{i}"] = np.array(step)
        out[f"stats_names{i}"] = np.array(list(stats))
        out[f"stats_text{i}"] = np.array(list(stats.values()))
        print(kws, {k: v.count("\n") for k, v in stats.items()})
    dst = os.path.join(ROOT, "tests", "golden", "det_ctc.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
