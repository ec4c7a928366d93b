#!/usr/bin/env python
"""Golden vectors for the streaming keyword spotter (test infrastructure): drives the REFERENCE's own
wekws/bin/stream_kws_ctc.py KeyWordSpotter (accept_wave + forward, chunk by chunk) with its model replaced by a module
that returns scripted logits -- peaky sequences that spell the keywords, built as make_ctc_golden.py builds them -- and
stores, per case, the chunk lengths, the frame count and PCM remainder after each chunk, the features accept_wave returned (first FEAT_CHUNKS chunks), the probabilities
the reference computed, every forward() return value and the final cur_hyps, in tests/golden/spotter.npz.
The reference's log is captured and every detection branch must have happened at least once.
      python oracle/make_spotter_golden.py"""
import logging
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFERENCE = "/root/reference"

V = 48
KEYWORDS = {"hi_xiaowen": [5, 9, 17, 23], "nihao_wenwen": [31, 7, 23, 23]}
FEAT_CHUNKS = 8
# front-ends: FSMN-CTC (80 mel, context 2/2, skip 3) and DS-TCN-CTC (40 mel, no context, skip 1)
CASES = [
    dict(name="fsmn", mel=80, context=(2, 2), skip=3, seed=11, threshold=0.5, min_frames=10, max_frames=120,
         interval_frames=100),
    dict(name="dstcn", mel=40, context=None, skip=1, seed=12, threshold=0.5, min_frames=5, max_frames=120,
         interval_frames=50),
]


def import_reference():
    """wekws.bin.stream_kws_ctc with the two modules this snapshot cannot provide stubbed: librosa (only its demo uses
    it) and the token / lexicon helpers of tools.make_list (not defined here; only set_keywords uses them)."""
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    sys.modules.setdefault("librosa", types.ModuleType("librosa"))
    import tools.make_list as ml
    for name in ("query_token_set", "read_lexicon", "read_token"):
        if not hasattr(ml, name):
            setattr(ml, name, None)
    import wekws.bin.stream_kws_ctc as S
    return S


def reference_spotter(S, model, mel, context, skip, threshold=0.0, min_frames=5, max_frames=250, interval_frames=50,
                      score_beam=3, path_beam=20):
    """A KeyWordSpotter with the fields __init__ / set_keywords would set (stream_kws_ctc.py:239-333), built without
    reading files."""
    k = object.__new__(S.KeyWordSpotter)
    torch.nn.Module.__init__(k)
    k.sample_rate, k.num_mel_bins, k.frame_length, k.frame_shift = 16000, mel, 25, 10
    k.downsampling, k.resolution = skip, 10 / 1000
    k.context_expansion = context is not None
    k.left_context, k.right_context = (0, 0) if context is None else context
    k.feats_ctx_offset = 0
    k.device = torch.device("cpu")
    k.model = model
    k.score_beam, k.path_beam = score_beam, path_beam
    k.threshold, k.min_frames, k.max_frames, k.interval_frames = threshold, min_frames, max_frames, interval_frames
    k.keywords_idxset = {0}.union(*[set(v) for v in KEYWORDS.values()])
    # token ids as a tuple, as score_ctc.py:168 builds them: is_sublist compares an equal-length prefix (a tuple) with ==
    k.keywords_token = {w: {"token_id": tuple(v)} for w, v in KEYWORDS.items()}
    k.reset_all()
    return k


class ScriptedModel(torch.nn.Module):
    """Returns the next T rows of a fixed logit sequence; the cache passes through."""

    def __init__(self, logits):
        super().__init__()
        self.logits, self.pos = logits, 0

    def forward(self, x, cache):
        T = x.size(1)
        out = self.logits[self.pos:self.pos + T].unsqueeze(0)
        assert out.size(1) == T, "scripted logits exhausted"
        self.pos += T
        return out, cache


def scripted_logits(T, seed, ds, max_frames):
    """Peaky CTC-like logits (random noise, an occasional competitor above the 0.05 gate) spelling, over and over: a
    keyword (activated), another one right after it (rejected by interval), silence until the dangling hypothesis is
    older than max_frames (reset), a weakly spelled keyword (rejected by threshold), silence, a keyword spelled in one
    frame per token (rejected by duration), silence.  `ds`: the model's frame skip, so the silences span max_frames."""
    g = torch.Generator().manual_seed(seed)
    a, b = list(KEYWORDS.values())
    silence = max_frames // ds + 8
    chunk = 30 // ds + 2               # the rest of the chunk after an activation is skipped (stream_kws_ctc.py:495-501)
    pattern = [(a, 2, 1, 9.0, chunk), (b, 2, 1, 9.0, silence), (a, 2, 1, 4.5, silence), (a, 1, 0, 9.0, silence)]
    logits = torch.randn(T, V, generator=g) * 0.3
    dom = torch.zeros(T, dtype=torch.long)
    sharp = torch.full((T,), 9.0)
    t, i = 2, 0
    while t < T:
        seq, reps, gap, strength, after = pattern[i % len(pattern)]
        for tok in seq:
            for _ in range(reps):
                if t < T:
                    dom[t], sharp[t] = tok, strength
                    t += 1
            t += gap
        t += after
        i += 1
    for t in range(T):
        logits[t, dom[t]] += float(sharp[t])
        if torch.rand(1, generator=g) < 0.1:
            logits[t, int(torch.randint(0, V, (1,), generator=g))] += float(sharp[t]) - 3.0
    return logits


def chunk_lengths(seed, context):
    """0.3 s chunks, odd sizes, chunks below the 800-sample hold, zero-length chunks and chunks that yield 3 frames.
    Without context expansion the reference raises on a buffer shorter than one window, so every chunk there has at
    least 400 samples."""
    rng = np.random.RandomState(seed)
    if context:
        lens = [4800, 4800, 1, 4800, 300, 200, 400, 3333, 0, 720, 4801, 560, 4800]
    else:
        lens = [4800, 4800, 401, 4800, 559, 720, 3333, 800, 4801, 400, 4800]
    lo = 0 if context else 400
    while len(lens) < (60 if context else 36):
        lens.append(int(rng.choice([4800, 4800, 4800, int(rng.randint(lo, 6000)), int(rng.randint(lo, 900))])))
    return np.array(lens, dtype=np.int64)


def case_pcm(seed, n):
    return np.random.RandomState(seed + 1000).randint(-3000, 3001, size=n).astype(np.int16)


def encode_result(r, words):
    """{} -> state -1; else (state, keyword index or -1, start, end, score) with NaN for None."""
    if not r:
        return -1, -1, np.nan, np.nan, np.nan
    if r["state"] == 1:
        return 1, words.index(r["keyword"]), r["start"], r["end"], r["score"]
    return 0, -1, np.nan, np.nan, np.nan


class _Log(logging.Handler):
    def __init__(self):
        super().__init__(logging.INFO)
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def run_case(S, c):
    lens = chunk_lengths(c["seed"], c["context"])
    pcm = case_pcm(c["seed"], int(lens.sum()))
    model = ScriptedModel(scripted_logits(4000, c["seed"], c["skip"], c["max_frames"]))
    k = reference_spotter(S, model, c["mel"], c["context"], c["skip"], c["threshold"], c["min_frames"],
                          c["max_frames"], c["interval_frames"])
    resets = []
    plain_reset = k.reset

    def reset():                       # activated is still True on the activation reset, False on the max_frames one
        resets.append("activation" if k.activated else "max_frames")
        plain_reset()
    k.reset = reset
    accept = k.accept_wave
    feats_seen = []

    def accept_wave(wave):
        f = accept(wave)
        feats_seen.append(None if f is None else f.clone())
        return f
    k.accept_wave = accept_wave
    words = list(KEYWORDS)
    out = {}
    frames, rems, feats, probs, results = [], [], [], [], []
    pos = 0
    for i, n in enumerate(lens):
        chunk = pcm[pos:pos + n]
        pos += n
        p0 = model.pos
        r = k.forward(chunk.tobytes())
        f = feats_seen[-1]
        frames.append(-1 if f is None else f.size(0))
        rems.append(len(k.wave_remained))
        if f is not None and i < FEAT_CHUNKS:
            feats.append(f.numpy().astype(np.float32))
        if model.pos > p0:                # the reference's own softmax of what the model returned
            probs.append(model.logits[p0:model.pos].softmax(1).numpy())
        results.append(encode_result(r, words))
    res = np.array(results, dtype=np.float64)
    hyps = k.cur_hyps
    L = max([len(h[0]) for h in hyps] + [1])
    tok = -np.ones((len(hyps), L), dtype=np.int32)
    frm = -np.ones((len(hyps), L), dtype=np.int32)
    prb = np.zeros((len(hyps), L), dtype=np.float64)
    for j, (prefix, (pb, pnb, nodes)) in enumerate(hyps):
        for q, nd in enumerate(nodes):
            tok[j, q], frm[j, q], prb[j, q] = prefix[q], nd["frame"], nd["prob"]
    out.update(lens=lens, frames=np.array(frames, dtype=np.int64), rem=np.array(rems, dtype=np.int64),
               feats=np.concatenate(feats) if feats else np.zeros((0, 1), np.float32),
               probs=np.concatenate(probs).astype(np.float32), result=res,
               hyp_len=np.array([len(h[0]) for h in hyps], dtype=np.int32), hyp_tok=tok, hyp_frame=frm, hyp_prob=prb,
               hyp_pb=np.array([h[1][0] for h in hyps]), hyp_pnb=np.array([h[1][1] for h in hyps]),
               pcm_sum=np.array(int(pcm.astype(np.int64).sum())))
    return out, resets


def main():
    S = import_reference()
    log = _Log()
    logging.getLogger().addHandler(log)
    logging.getLogger().setLevel(logging.INFO)
    out = {"V": np.array(V), "ncases": np.array(len(CASES)), "feat_chunks": np.array(FEAT_CHUNKS),
           "kw_names": np.array(list(KEYWORDS)), "kw_tokens": np.array([t for v in KEYWORDS.values() for t in v]),
           "kw_offsets": np.cumsum([0] + [len(v) for v in KEYWORDS.values()])}
    all_resets = []
    for i, c in enumerate(CASES):
        got, resets = run_case(S, c)
        all_resets += resets
        for k, v in got.items():
            out[f"{k}{i}"] = v
        for k in ("mel", "skip", "seed", "threshold", "min_frames", "max_frames", "interval_frames"):
            out[f"{k}{i}"] = np.array(c[k])
        out[f"context{i}"] = np.array(c["context"] if c["context"] else (0, 0))
        print(c["name"], "chunks", len(got["lens"]), "model frames", len(got["probs"]), "activations",
              int((got["result"][:, 0] == 1).sum()), "resets", {r: resets.count(r) for r in set(resets)})
    text = "\n".join(log.lines)
    branches = {"activated": "Activated." in text, "interval": "but interval" in text,
                "threshold": "is lower than 0.5, Deactivated" in text, "duration": "beyond range" in text,
                "max_frames reset": "max_frames" in all_resets}
    print(branches)
    assert all(branches.values()), f"a detection branch never happened: {branches}"
    dst = os.path.join(ROOT, "tests", "golden", "spotter.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, os.path.getsize(dst), "bytes")


if __name__ == "__main__":
    main()
