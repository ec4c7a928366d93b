#!/usr/bin/env python
"""Golden vectors for the streaming CTC scorer (test infrastructure): runs the REFERENCE's own
wekws/bin/stream_score_ctc.py main() in-process on scripted posteriors and stores, per configuration, the posteriors it
decoded (its own CPU softmax), the lengths, keys and arguments, the score file it wrote and every "detect ... from S to
E ..." log record, parsed, in tests/golden/stream_score.npz.

The snapshot cannot import wenet, so wenet.text.char_tokenizer (a character -> id tokenizer) and wenet.dataset.dataset
are stub modules, and init_dataset / DataLoader / init_model / load_checkpoint are replaced in the script's namespace:
the loader yields scripted padded batches and the model returns scripted logits.  --gpu -1 runs it on the CPU.
Every detection branch must have happened at least once.
      python oracle/make_stream_score_golden.py"""
import logging
import os
import re
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFERENCE = "/root/reference"

V = 32
CHARS = {"a": 5, "b": 9, "c": 17, "d": 23, "e": 29, "f": 7}     # the stub tokenizer's dictionary; others -> 1
KEYWORDS = "abcd,efdd"
EMPTY_TOKEN = 30                                                 # outside the keyword set: its frames are filtered out
CONFIGS = [
    dict(name="skip1", frame_skip=1, threshold=0.0, min_frames=5, max_frames=60, score_beam=3, path_beam=20, seed=21,
         batches=[5, 4, 3]),
    dict(name="skip3", frame_skip=3, threshold=0.5, min_frames=10, max_frames=90, score_beam=3, path_beam=20, seed=22,
         batches=[4, 5, 3]),
]


def keyword_tokens():
    """{word: token ids} as the script builds them (:191-199), in --keywords order."""
    return {w: [CHARS.get(ch, 1) for ch in w] for w in KEYWORDS.split(",")}


class CharTokenizer:
    def __init__(self, *args, **kwargs):
        pass

    def tokenize(self, line):
        strs = line.split(" ")
        return strs, [CHARS.get(s, 1) for s in strs]


def import_reference():
    """wekws.bin.stream_score_ctc with the wenet modules it imports stubbed."""
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    for name in ("wenet", "wenet.text", "wenet.dataset"):
        sys.modules.setdefault(name, types.ModuleType(name))
    tok = types.ModuleType("wenet.text.char_tokenizer")
    tok.CharTokenizer = CharTokenizer
    sys.modules["wenet.text.char_tokenizer"] = tok
    ds = types.ModuleType("wenet.dataset.dataset")
    ds.Dataset = object
    sys.modules["wenet.dataset.dataset"] = ds
    import wekws.bin.stream_score_ctc as S
    return S


# ---------------------------------------------------------------------------------------------------------- scripts
def _segment(kind, kw, rng):
    """(token, strength) rows of one scripted segment; token None = noise only, strength is added to its logit."""
    toks = keyword_tokens()[kw] if kw else []
    rows = []
    if kind == "strong":            # 2 frames per token, a blank between tokens
        for t in toks:
            rows += [(t, 9.0)] * 2 + [(0, 9.0)]
    elif kind == "weak":            # each token at ~0.3 under a ~0.6 blank: the keyword is not the first hypothesis
        for t in toks:
            rows += [("weak", t)] * 2 + [(0, 9.0)]
    elif kind == "fast":            # one frame per token: too short
        rows += [(t, 9.0) for t in toks]
    elif kind == "slow":            # long blanks between tokens: too long
        for t in toks:
            rows += [(t, 9.0)] * 2 + [(0, 9.0)] * int(rng.randint(24, 32))
    elif kind == "empty":           # frames whose top-k is filtered out entirely
        rows += [(EMPTY_TOKEN, 9.0)] * int(rng.randint(2, 8))
    elif kind == "silence":
        rows += [(0, 9.0)] * int(rng.randint(3, 12))
    return rows


def utterance_logits(program, rng, noise=0.3):
    rows = []
    for kind, kw in program:
        rows += _segment(kind, kw, rng)
    x = torch.from_numpy(rng.randn(len(rows), V).astype(np.float32)) * noise
    for t, (tok, s) in enumerate(rows):
        if tok == "weak":
            x[t, 0] += 7.0
            x[t, s] += 6.3
        else:
            x[t, tok] += s
        if rng.rand() < 0.1:        # an occasional competitor above the 0.05 gate
            x[t, int(rng.randint(0, V))] += 6.0
    return x


HAND = [
    [("silence", None), ("strong", "abcd"), ("silence", None), ("empty", None), ("strong", "efdd"), ("silence", None)],
    [("silence", None), ("weak", "abcd"), ("silence", None), ("silence", None), ("silence", None)],
    [("silence", None), ("fast", "abcd"), ("silence", None), ("empty", None), ("silence", None)],
    [("silence", None), ("slow", "efdd"), ("silence", None)],
    [],
    [("empty", None), ("silence", None), ("empty", None)],
    [("strong", "efdd"), ("empty", None), ("weak", "efdd"), ("silence", None), ("strong", "abcd"), ("silence", None)],
]
KINDS = ["strong", "weak", "fast", "slow", "empty", "silence", "silence"]


def random_program(rng):
    n = int(rng.randint(0, 7))
    out = []
    for _ in range(n):
        kind = KINDS[int(rng.randint(len(KINDS)))]
        out.append((kind, None if kind in ("empty", "silence") else ["abcd", "efdd"][int(rng.randint(2))]))
    return out


def make_batches(sizes, seed, hand=True, max_rows=None):
    """[(keys, padded logits (b, T, V), lengths (b,))]; the first utterances follow HAND, the rest are random."""
    rng = np.random.RandomState(seed)
    progs = list(HAND) if hand else []
    batches, u = [], 0
    for bi, n in enumerate(sizes):
        xs = []
        for _ in range(n):
            prog = progs[u] if u < len(progs) else random_program(rng)
            x = utterance_logits(prog, rng)
            if max_rows is not None:
                x = x[:max_rows]
            xs.append(x)
            u += 1
        T = max([x.shape[0] for x in xs] + [1]) + int(rng.randint(0, 4))     # padding past the longest
        pad = torch.from_numpy(rng.randn(n, T, V).astype(np.float32))
        for i, x in enumerate(xs):
            pad[i, :x.shape[0]] = x
        keys = [f"utt{seed}_{bi}_{i}" for i in range(n)]
        batches.append((keys, pad, torch.tensor([x.shape[0] for x in xs], dtype=torch.int64)))
    return batches


# ---------------------------------------------------------------------------------------------------------- driver
class _Log(logging.Handler):
    def __init__(self):
        super().__init__(logging.DEBUG)
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


_DETECT = re.compile(r"^batch:(\d+)_(\d+) detect (\S+) in (\S+) from (-?\d+) to (-?\d+) frame\. (.*)$")
ACTIVATED, LOW_SCORE, BAD_DURATION = 0, 1, 2


def parse_records(lines):
    """The detect log lines -> [(key, kind, keyword, score or nan, start, end)]."""
    out = []
    for line in lines:
        m = _DETECT.match(line)
        if m is None:
            continue
        key, kw, start, end, rest = m.group(4), m.group(3), int(m.group(5)), int(m.group(6)), m.group(7)
        if rest.endswith("Activated."):
            kind, score = ACTIVATED, float(re.search(r"score (\S+) Activated\.$", rest).group(1))
        elif "less than" in rest:
            kind, score = LOW_SCORE, float(re.match(r"but (\S+) less than", rest).group(1))
        else:
            assert "beyond range" in rest, line
            kind, score = BAD_DURATION, float("nan")
        out.append((key, kind, kw, score, start, end))
    return out


def run_reference(S, cfg, batches):
    """Runs main() over the batches -> (score-file text, parsed detect records, [(keys, probs, lengths)] decoded)."""
    decoded = []

    class Model(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.i = 0

        def forward(self, feats):
            logits = batches[self.i][1]
            assert feats.shape[:2] == logits.shape[:2]
            self.i += 1
            decoded.append(logits.softmax(2))          # what the script computes from it (:219)
            return logits, None

    def init_dataset(**kwargs):
        return [dict(keys=k, feats=torch.zeros(x.shape[0], x.shape[1], 1), target=torch.ones(x.shape[0], 1,
                     dtype=torch.long), feats_lengths=n, target_lengths=torch.ones(x.shape[0], dtype=torch.long))
                for k, x, n in batches]

    S.init_dataset = init_dataset
    S.DataLoader = lambda ds, **kwargs: ds
    S.init_model = lambda conf: Model()
    S.load_checkpoint = lambda model, path: {}
    log = _Log()
    root = logging.getLogger()
    old_level = root.level
    root.addHandler(log)
    root.setLevel(logging.DEBUG)
    with tempfile.TemporaryDirectory() as tmp:
        conf = os.path.join(tmp, "conf.yaml")
        with open(conf, "w") as f:
            f.write("dataset_conf:\n  filter_conf: {}\n  fbank_conf: {}\n  batch_conf: {}\n"
                    f"  frame_skip: {cfg['frame_skip']}\nmodel: {{}}\n")
        score = os.path.join(tmp, "score.txt")
        argv = sys.argv
        sys.argv = ["stream_score_ctc.py", "--config", conf, "--test_data", "unused", "--checkpoint", "unused",
                    "--gpu", "-1", "--score_file", score, "--keywords", KEYWORDS,
                    "--score_beam_size", str(cfg["score_beam"]), "--path_beam_size", str(cfg["path_beam"]),
                    "--threshold", str(cfg["threshold"]), "--min_frames", str(cfg["min_frames"]),
                    "--max_frames", str(cfg["max_frames"])]
        try:
            S.main()
        finally:
            sys.argv = argv
            root.removeHandler(log)
            root.setLevel(old_level)
        with open(score, encoding="utf8") as f:
            text = f.read()
    return text, parse_records(log.lines), [(k, p, n) for (k, _, n), p in zip(batches, decoded)]


def branches(cfg, text, records, decoded):
    """Which detection branches the run took (checked on the reference's own output and the oracle's frames)."""
    from oracle.kws_stream_score_oracle import stream_score
    kws = keyword_tokens()
    got = dict(activation=False, second_activation=False, low_score=False, too_short=False, too_long=False,
               empty_between_hits=False, late_activation=False, never_activated="rejected" in text,
               zero_length=False)
    acts = {}
    for i, (key, kind, kw, score, start, end) in enumerate(records):
        d = end - start
        got["activation"] |= kind == ACTIVATED
        got["low_score"] |= kind == LOW_SCORE
        got["too_short"] |= kind == BAD_DURATION and d < cfg["min_frames"]
        got["too_long"] |= kind == BAD_DURATION and d > cfg["max_frames"]
        if kind == ACTIVATED:
            acts[key] = acts.get(key, 0) + 1
            prev = records[i - 1] if i else None
            # quirk 2: the first hypothesis lost the keyword, sqrt raised the stale score, the stale hit fired
            got["late_activation"] |= (prev is not None and prev[0] == key and prev[1] == LOW_SCORE
                                       and prev[2:3] + prev[4:] == (kw, start, end) and prev[3] < score)
    got["second_activation"] = any(n >= 2 for n in acts.values())
    from oracle.kws_stream_score_oracle import _decoded
    tokenset = {0}.union(*[set(s) for s in kws.values()])
    for keys, probs, lens in decoded:
        for b, key in enumerate(keys):
            n = int(lens[b])
            got["zero_length"] |= n == 0
            _, events = stream_score(probs[b, :n], kws, cfg["score_beam"], cfg["path_beam"], cfg["threshold"],
                                     cfg["min_frames"], cfg["max_frames"], cfg["frame_skip"])
            frames = [e[5] // cfg["frame_skip"] for e in events]
            for lo, hi in zip(frames, frames[1:]):
                if any(not _decoded(probs[b, t], tokenset, cfg["score_beam"]) for t in range(lo + 1, hi)):
                    got["empty_between_hits"] = True
    return got


def main():
    S = import_reference()
    out = {"V": np.array(V), "nconfigs": np.array(len(CONFIGS)), "kw_names": np.array(list(keyword_tokens())),
           "kw_tokens": np.array([t for v in keyword_tokens().values() for t in v]),
           "kw_offsets": np.cumsum([0] + [len(v) for v in keyword_tokens().values()])}
    seen = {}
    for c, cfg in enumerate(CONFIGS):
        text, records, decoded = run_reference(S, cfg, make_batches(cfg["batches"], cfg["seed"]))
        got = branches(cfg, text, records, decoded)
        print(cfg["name"], got)
        for k, v in got.items():
            seen[k] = seen.get(k, False) or v
        # every utterance's valid rows, back to back (padding is not stored)
        keys = [k for ks, _, _ in decoded for k in ks]
        lens = np.concatenate([n.numpy() for _, _, n in decoded]).astype(np.int32)
        rows = np.concatenate([p[b, :int(n[b])].numpy() for _, p, n in decoded for b in range(len(n))])
        out[f"probs{c}"] = rows.astype(np.float32)
        out[f"lengths{c}"] = lens
        out[f"batch_sizes{c}"] = np.array(cfg["batches"], dtype=np.int32)
        out[f"keys{c}"] = np.array(keys)
        out[f"score_text{c}"] = np.array(text)
        out[f"rec_key{c}"] = np.array([r[0] for r in records])
        out[f"rec{c}"] = np.array([(r[1], keyword_index(r[2]), r[4], r[5]) for r in records], dtype=np.int32
                                  ).reshape(-1, 4)
        out[f"rec_score{c}"] = np.array([r[3] for r in records], dtype=np.float64)
        for k in ("frame_skip", "threshold", "min_frames", "max_frames", "score_beam", "path_beam"):
            out[f"{k}{c}"] = np.array(cfg[k])
    print(seen)
    assert all(seen.values()), f"a detection branch never happened: {seen}"
    dst = os.path.join(ROOT, "tests", "golden", "stream_score.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


def keyword_index(word):
    return list(keyword_tokens()).index(word)


if __name__ == "__main__":
    main()
