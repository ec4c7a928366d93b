#!/usr/bin/env python
"""Golden vectors for the training criteria (test infrastructure): runs the REFERENCE's own wekws/model/loss.py
criterion() and wekws/utils/executor.py Executor.cv on scripted batches on the CPU and writes
tests/golden/criterion.npz.

Per call <name>: the inputs, the reference's (loss, acc) or the exception it raised, and for ce / ctc the same loss
in float64 (the spread the device tolerances are derived from).  Per CTC call also the per-utterance losses
(reduction='none', float32 and float64), and with validation the reference's best hypotheses and Calculator results.
Per cv run <name>: the batches Executor.cv reads (dicts of keys / feats / target (B, Lmax) / feats_lengths /
target_lengths; the model returns feats as the logits) and its totals.

The device softmax is not bit-identical to torch's CPU softmax, so every decoded frame's top-3 probabilities are kept
at least 1e-5 away from the decoder's 0.05 filter and from each other and from the 4th (no top-k ties); this is
asserted.
      python oracle/make_criterion_golden.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REFERENCE = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "criterion.npz")
MARGIN = 1e-5


def import_reference():
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    from wekws.model import loss
    from wekws.utils import executor
    return loss, executor


def margins_ok(probs):
    """probs (n, V): top-3 away from 0.05 and no near-ties among the top 4."""
    top = probs.double().topk(min(4, probs.size(1)), dim=1)[0]
    if (top[:, :3] - 0.05).abs().min() < MARGIN:
        return False
    return bool((top[:, :-1] - top[:, 1:]).min() >= MARGIN)


def ctc_logits(rng, B, T, V, labels, lengths):
    """Peaky logits that mostly spell each label with blanks between tokens; every frame meets margins_ok."""
    x = torch.zeros(B, T, V)
    for b in range(B):
        lab = labels[b]
        n = int(lengths[b])
        path = []
        for tok in lab:
            path += [tok] * int(rng.integers(1, 3)) + [0] * int(rng.integers(0, 3))
        path = ([0] * int(rng.integers(0, 3)) + path + [0] * n)[:n] if n else []
        for t in range(T):
            while True:
                row = torch.from_numpy(rng.normal(0.0, 1.0, V).astype(np.float32))
                if t < n:
                    hot = path[t] if rng.random() < 0.9 else int(rng.integers(0, V))
                    row[hot] += float(rng.uniform(4.0, 8.0))
                    row[int(rng.integers(0, V))] += float(rng.uniform(0.0, 3.0))
                if t >= n or margins_ok(row.softmax(0)[None]):
                    break
            x[b, t] = row
    return x


def big_vocab_logits(rng, B, T, V, labels, lengths):
    """V = 2599 logits that compress: a quantised background and a few raised tokens per frame."""
    x = torch.from_numpy((rng.integers(-8, 8, size=(B, T, V)) * 0.25).astype(np.float32))
    for b in range(B):
        lab = labels[b]
        for t in range(int(lengths[b])):
            hot = lab[(t // 3) % len(lab)] if (lab and t % 3 != 2) else 0
            while True:                                  # three distinct raised tokens: the top 3 never tie
                row = x[b, t].clone()
                toks = [hot] + [int(v) for v in rng.choice(V, 2, replace=False)]
                if len(set(toks)) < 3:
                    continue
                for tok, lift in zip(toks, sorted(rng.choice(np.arange(12, 48), 3, replace=False), reverse=True)):
                    row[tok] = 2.0 + float(lift) * 0.25
                if margins_ok(row.softmax(0)[None]):
                    break
            x[b, t] = row
    return x


def padded(labels, width=None):
    width = width or max(1, max(len(l) for l in labels))
    t = torch.full((len(labels), width), -1, dtype=torch.int64)
    for b, l in enumerate(labels):
        t[b, :len(l)] = torch.tensor(l, dtype=torch.int64)
    return t, torch.tensor([len(l) for l in labels], dtype=torch.int64)


def mp_case(rng, B, T, D, targets, lengths, nan=False, tie=False):
    x = torch.from_numpy(rng.uniform(0.0, 1.0, size=(B, T, D)).astype(np.float32))
    x = x ** 3                                           # mostly low posteriors, so some maxima fall below 0.5
    if tie:                                              # utterance 0: two keyword columns share the highest value
        x[0, 3, 0] = x[0, 5, 1] = 0.96875
        x[0, :, :] = x[0].clamp(max=0.9)
        x[0, 3, 0] = x[0, 5, 1] = 0.96875
    if nan:
        x[1, 2, 0] = float("nan")                        # a NaN in a valid frame propagates
        x[2, T - 1, 1] = float("nan")                    # a NaN in a padding frame is masked away
    return x, torch.tensor(targets, dtype=torch.int64), torch.tensor(lengths, dtype=torch.int64)


def run(fn):
    try:
        return fn(), None
    except Exception as e:                               # the reference's own failure is part of the contract
        return None, type(e).__name__


def main():
    loss_mod, executor = import_reference()
    rng = np.random.default_rng(2024)
    g = {}

    def put(name, **kw):
        for k, v in kw.items():
            g[f"{name}__{k}"] = v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v)

    def call(name, ctype, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
        res, err = run(lambda: loss_mod.criterion(ctype, logits, target, lengths, target_lengths, min_duration,
                                                  validation))
        put(name, type=ctype, logits=logits, target=target, min_duration=min_duration, validation=int(validation),
            error=err or "")
        if lengths is not None:
            put(name, lengths=lengths)
        if target_lengths is not None:
            put(name, target_lengths=target_lengths)
        if res is not None:
            loss, acc = res
            put(name, loss=np.float32(loss.item()), acc=np.float64(acc))
        if ctype == "ce" and res is not None:
            put(name, loss64=np.float64(torch.nn.functional.cross_entropy(logits.double(), target.long()).item()))
        if ctype == "ctc" and res is not None:
            lp = logits.transpose(0, 1).log_softmax(2)
            put(name, utt_loss=torch.nn.functional.ctc_loss(lp, target, lengths, target_lengths, reduction="none"),
                utt_loss64=torch.nn.functional.ctc_loss(lp.double(), target, lengths, target_lengths,
                                                        reduction="none"),
                loss64=np.float64((torch.nn.functional.ctc_loss(lp.double(), target, lengths, target_lengths,
                                                                 reduction="sum") / lp.size(1)).item()))
            if validation and target.dim() == 2:
                decode_details(name, logits, target, lengths, target_lengths)
        names.append(name)

    def decode_details(name, logits, target, lengths, target_lengths):
        """acc_utterance's loop (loss.py:113-129) with its intermediate results kept."""
        probs = logits.softmax(2)
        calc = loss_mod.Calculator()
        hyp = np.full((logits.size(0), 1 + 64), -1, dtype=np.int32)
        res = np.zeros((logits.size(0), 5), dtype=np.int64)        # all, cor, sub, ins, del
        for i in range(logits.size(0)):
            n = int(lengths[i])
            assert margins_ok(probs[i][:n]) if n else True
            hyps = loss_mod.ctc_prefix_beam_search(probs[i][:n], lengths[i], None, 3, 5)
            rec = list(hyps[0][0]) if hyps else []
            hyp[i, 0] = len(rec)
            hyp[i, 1:1 + len(rec)] = rec
            r = calc.calculate([str(v) for v in target[i][:int(target_lengths[i])].tolist()], [str(v) for v in rec])
            res[i] = [r["all"], r["cor"], r["sub"], r["ins"], r["del"]]
        put(name, best=hyp, calc=res)

    names = []
    # ---- max_pooling: fillers (-1, -3), out-of-range keyword targets (2, 7), padded lengths, ties, NaN
    D, T = 2, 24
    x, t, l = mp_case(rng, 8, T, D, [1, 0, -1, 2, 0, -3, 7, 1], [24, 20, 11, 24, 3, 17, 24, 9], tie=True)
    call("mp0", "max_pooling", x, t, l)
    call("mp0_dur", "max_pooling", x, t, l, min_duration=6)
    x, t, l = mp_case(rng, 6, T, D, [0, 1, -1, 0, 1, -1], [24, 24, 20, 13, 24, 1], nan=True)
    call("mp1_nan", "max_pooling", x, t, l)
    x, t, l = mp_case(rng, 5, 30, 3, [2, -1, 0, 1, -1], [30, 29, 30, 7, 22])
    call("mp2", "max_pooling", x, t, l, min_duration=3)
    # ---- ce: -100 rows, argmax ties, an out-of-range target (IndexError), all ignored (nan)
    Cn = 12
    x = torch.from_numpy(rng.normal(0, 2, size=(10, Cn)).astype(np.float32))
    x[3, 4] = x[3, 9] = x[3].max() + 1.0                # tie: the first index wins
    x[5, 0] = x[5, 7] = x[5].max() + 1.0
    t = torch.tensor([4, -100, 2, 9, 11, 0, -100, 5, 5, 1])
    call("ce0", "ce", x, t, None)
    call("ce_all_ignored", "ce", x[:3], torch.tensor([-100, -100, -100]), None)
    call("ce_bad_target", "ce", x[:3], torch.tensor([1, 12, 0]), None)
    x = torch.from_numpy(rng.normal(0, 3, size=(7, 3)).astype(np.float32))
    call("ce1", "ce", x, torch.tensor([0, 1, 2, 2, 1, 0, 1]), None)
    # ---- ctc, V = 32: repeated labels, an empty label, an infeasible utterance (T_b < L_b + repeats)
    V, T = 32, 40
    labels = [[3, 3, 7], [5, 9, 12, 5], [], [8, 8, 8], [20, 4], [6, 1, 1, 2, 30]]
    lens = torch.tensor([40, 33, 12, 4, 40, 25])            # utterance 3: 3 tokens + 2 repeats > 4 frames
    tgt, tl = padded(labels)
    x = ctc_logits(rng, len(labels), T, V, labels, lens)
    call("ctc0", "ctc", x, tgt, lens, tl, validation=True)
    call("ctc0_loss", "ctc", x, tgt, lens, tl, validation=False)
    labels1 = [[3, 3, 7], [5, 9, 12, 5], [], [8, 8, 8, 2, 2], [20, 4], [6, 1, 1, 2, 30], [17], [11, 11, 11, 11]]
    lens1 = torch.tensor([40, 38, 12, 30, 40, 25, 9, 21])
    tgt1, tl1 = padded(labels1)
    x1 = ctc_logits(rng, len(labels1), T, V, labels1, lens1)
    call("ctc1", "ctc", x1, tgt1, lens1, tl1, validation=True)
    # the 1-D target Executor.cv makes when Lmax == 1: F.ctc_loss reads concatenated labels; acc_utterance cannot index it
    labels2 = [[4], [9], [0 + 13], [2]]
    lens2 = torch.tensor([10, 16, 7, 16])
    x2 = ctc_logits(rng, 4, 16, V, labels2, lens2)
    tgt2 = torch.tensor([4, 9, 13, 2])
    tl2 = torch.ones(4, dtype=torch.int64)
    call("ctc_1d", "ctc", x2, tgt2, lens2, tl2, validation=False)
    call("ctc_1d_val", "ctc", x2, tgt2, lens2, tl2, validation=True)
    # every label empty: acc_utterance divides by zero
    tge, tle = padded([[], [], []], width=2)
    call("ctc_empty", "ctc", x2[:3], tge, lens2[:3], tle, validation=True)
    call("ctc_empty_loss", "ctc", x2[:3], tge, lens2[:3], tle, validation=False)
    # ---- ctc, V = 2599 (the shipped vocabulary), small
    V3, T3 = 2599, 14
    labels3 = [[1021, 77, 77, 2598], [5, 1800]]
    lens3 = torch.tensor([14, 11])
    tgt3, tl3 = padded(labels3)
    x3 = big_vocab_logits(rng, 2, T3, V3, labels3, lens3)
    call("ctc_v2599", "ctc", x3, tgt3, lens3, tl3, validation=True)

    # ---- Executor.cv over scripted loaders
    class Echo(torch.nn.Module):                         # the model returns its input as the logits
        def forward(self, feats):
            return feats, None

    def cv_run(name, ctype, batches):
        args = {"criterion": ctype, "log_interval": 1000}
        loss, acc = executor.Executor().cv(Echo(), batches, torch.device("cpu"), args)
        put(name, type=ctype, nbatch=len(batches), loss=np.float64(loss), acc=np.float64(acc))
        for k, bd in enumerate(batches):
            put(f"{name}_b{k}", **{key: bd[key] for key in ("feats", "target", "feats_lengths", "target_lengths")})
        cvs.append(name)

    def batch(feats, target2d, lengths, target_lengths):
        return {"keys": [f"utt{i}" for i in range(feats.size(0))], "feats": feats, "target": target2d,
                "feats_lengths": lengths, "target_lengths": target_lengths}

    cvs = []
    mp = [(g[f"{n}__logits"], g[f"{n}__target"], g[f"{n}__lengths"]) for n in ("mp0", "mp1_nan", "mp2")]
    cv_run("cv_mp", "max_pooling",
           [batch(torch.from_numpy(x), torch.from_numpy(t)[:, None], torch.from_numpy(l), torch.ones(len(l),
                                                                                                   dtype=torch.int64))
            for x, t, l in mp[:2]])                     # mp1_nan's loss is NaN: the batch is skipped
    ce_x = torch.from_numpy(g["ce0__logits"])
    ce_t = torch.tensor([4, 3, 2, 9, 11, 0, 1, 5, 5, 1])
    cv_run("cv_ce", "ce", [batch(ce_x[:6], ce_t[:6, None], torch.ones(6, dtype=torch.int64),
                                 torch.ones(6, dtype=torch.int64)),
                           batch(ce_x[6:], ce_t[6:, None], torch.ones(4, dtype=torch.int64),
                                 torch.ones(4, dtype=torch.int64))])
    cv_run("cv_ctc", "ctc", [batch(x, tgt, lens, tl), batch(x1, tgt1, lens1, tl1)])   # the first batch is inf: skipped

    g["names"] = np.array(names)
    g["cv_names"] = np.array(cvs)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(names)} calls, {len(cvs)} cv runs")
    for n in names:
        print(n, g[f"{n}__error"] or (float(g[f"{n}__loss"]), float(g[f"{n}__acc"])))
    for n in cvs:
        print(n, float(g[f"{n}__loss"]), float(g[f"{n}__acc"]))


if __name__ == "__main__":
    main()
