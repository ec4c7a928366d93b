#!/usr/bin/env python
"""Golden gradients of the training criteria (test infrastructure): differentiates the REFERENCE's own
wekws/model/loss.py criterion() with torch's autograd on the CPU, as Executor.train does (loss.backward()), in float32
and in float64, and writes tests/golden/criterion_grad.npz.

Per call <name>: the inputs, the upstream gradient `up` (the loss is multiplied by it before backward()), the loss and
d (up * loss) / d logits in float32 (`loss`, `grad`) and float64 (`loss64`, `grad64`).  The cases cover what the
device kernels must reproduce: max-pooling ties (split evenly, masked and out-of-clamp ties counted but not paid),
min_duration, the clamp's closed ends, fillers and targets >= D, NaN posteriors; cross entropy with ignored rows and
with every row ignored; CTC with repeated tokens, an empty label, an utterance of no frames, an infeasible utterance
shorter than T (NaN rows), 1-D targets, the shipped vocabulary of 2599 tokens; upstream gradients other than 1.
      python oracle/make_criterion_grad_golden.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_criterion_golden import import_reference, padded  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "criterion_grad.npz")


def main():
    loss_mod, _ = import_reference()
    rng = np.random.default_rng(4242)
    g, names = {}, []

    def grad_of(ctype, logits, target, lengths, target_lengths, min_duration, up, dtype):
        x = logits.detach().to(dtype).clone().requires_grad_(True)
        loss, _ = loss_mod.criterion(ctype, x, target, lengths, target_lengths, min_duration, False)
        (loss * up).backward()
        return loss.detach(), x.grad

    def call(name, ctype, logits, target, lengths=None, target_lengths=None, min_duration=0, up=1.0):
        l32, g32 = grad_of(ctype, logits, target, lengths, target_lengths, min_duration, up, torch.float32)
        l64, g64 = grad_of(ctype, logits, target, lengths, target_lengths, min_duration, up, torch.float64)
        rec = dict(type=ctype, logits=logits, target=target, min_duration=min_duration, up=np.float32(up),
                   loss=np.float32(l32.item()), grad=g32, loss64=np.float64(l64.item()), grad64=g64)
        if lengths is not None:
            rec["lengths"] = lengths
        if target_lengths is not None:
            rec["target_lengths"] = target_lengths
        for k, v in rec.items():
            g[f"{name}__{k}"] = v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        names.append(name)

    # ---- max_pooling.  utterance 0: keyword column [1, 1, .5, 1] and a two-way tie of the other column's minimum;
    # utterance 1: filler whose padded frame would tie; utterance 2: target >= D, posteriors 0 (1 - p ties at the
    # clamp's upper end with the padding's fill value); utterance 3: keyword column 1 with a tie across min_duration
    x = torch.tensor([[[1.0, 0.2], [1.0, 0.7], [0.5, 0.7], [1.0, 0.1]],
                      [[0.9, 0.3], [0.9, 0.3], [0.3, 0.1], [0.9, 0.3]],
                      [[0.0, 0.0], [0.0, 0.25], [0.6, 0.9], [0.6, 0.9]],
                      [[0.1, 0.75], [0.2, 0.75], [0.1, 0.25], [0.2, 0.75]]])
    t = torch.tensor([0, -1, 5, 1])
    l = torch.tensor([4, 3, 2, 4])
    call("mp_ties", "max_pooling", x, t, l)
    call("mp_ties_dur2", "max_pooling", x, t, l, min_duration=2)
    call("mp_ties_up3", "max_pooling", x, t, l, up=3.0)
    # the clamp's ends: keyword column [1e-8, 0] (two-way tie at the lower end, half of it lost), keyword column
    # [0, 0] (every tie outside), other column of ones (1 - p = 0, outside) and [1, .5]
    x = torch.tensor([[[1e-8, 1.0], [0.0, 1.0]], [[1.0, 0.0], [0.5, 0.0]]])
    call("mp_clamp", "max_pooling", x, torch.tensor([0, 1]), torch.tensor([2, 2]))
    # random posteriors saturated to exact 0 / 1 in places, fillers (-1, -3), targets >= D, padding, a NaN
    x = torch.from_numpy(rng.uniform(0.0, 1.0, size=(8, 24, 2)).astype(np.float32)) ** 3
    x[torch.from_numpy(rng.random((8, 24, 2)) < 0.15)] = 1.0
    x[torch.from_numpy(rng.random((8, 24, 2)) < 0.10)] = 0.0
    t = torch.tensor([1, 0, -1, 2, 0, -3, 7, 1])
    l = torch.tensor([24, 20, 11, 24, 3, 17, 24, 9])
    call("mp_rand", "max_pooling", x, t, l)
    call("mp_rand_dur6", "max_pooling", x, t, l, min_duration=6, up=0.375)
    xn = x.clone()
    xn[1, 2, 0] = float("nan")                           # in the keyword column of utterance 1
    xn[2, 23, 1] = float("nan")                          # in a padding frame: masked away
    xn[3, 5, 1] = float("nan")                           # in an other column
    call("mp_nan", "max_pooling", xn, t, l)
    x3 = torch.from_numpy(rng.uniform(0.0, 1.0, size=(5, 30, 3)).astype(np.float32))
    call("mp_d3", "max_pooling", x3, torch.tensor([2, -1, 0, 1, -1]), torch.tensor([30, 29, 30, 7, 22]),
         min_duration=3)

    # ---- ce: ignored rows, every row ignored (loss NaN, gradient zeros), an upstream gradient
    x = torch.from_numpy(rng.normal(0, 2, size=(10, 12)).astype(np.float32))
    t = torch.tensor([4, -100, 2, 9, 11, 0, -100, 5, 5, 1])
    call("ce0", "ce", x, t)
    call("ce0_up3", "ce", x, t, up=3.0)
    call("ce_all_ignored", "ce", x[:3], torch.tensor([-100, -100, -100]))
    call("ce1", "ce", torch.from_numpy(rng.normal(0, 3, size=(7, 3)).astype(np.float32)),
         torch.tensor([0, 1, 2, 2, 1, 0, 1]))

    # ---- ctc, V = 9: repeats (adjacent and apart), an empty label, an empty label on no frames
    V, T = 9, 12
    labels = [[3, 3, 5], [1, 2, 1, 2], [], [7], [], [4, 6, 4, 4, 8]]
    lens = torch.tensor([12, 10, 5, 1, 0, 11])
    tgt, tl = padded(labels)
    x = torch.from_numpy(rng.normal(0, 2, size=(len(labels), T, V)).astype(np.float32))
    call("ctc0", "ctc", x, tgt, lens, tl)
    call("ctc0_up3", "ctc", x, tgt, lens, tl, up=3.0)
    # utterance 1 is infeasible (3 tokens + 2 repeats > 4 frames) and shorter than T; utterance 3 too (no frames)
    labels = [[3, 3, 5], [8, 8, 8], [2], [1, 2]]
    lens_inf = torch.tensor([12, 4, 9, 0])
    tgt_inf, tl_inf = padded(labels)
    call("ctc_infeasible", "ctc", x[:4], tgt_inf, lens_inf, tl_inf)
    # 1-D concatenated labels, as F.ctc_loss reads the target Executor makes when Lmax == 1
    call("ctc_1d", "ctc", x[:4], torch.tensor([4, 8, 1, 2]), torch.tensor([10, 12, 7, 3]),
         torch.ones(4, dtype=torch.int64))
    call("ctc_1d_ragged", "ctc", x[:3], torch.tensor([4, 4, 8, 1, 2, 1]), torch.tensor([10, 12, 7]),
         torch.tensor([2, 1, 3]))
    # V = 2599: rows of the logits and of the gradient start on every 4-byte phase of a 16-byte line
    labels = [[1021, 77, 2598], [5, 1800]]
    lens = torch.tensor([4, 3])
    tgt, tl = padded(labels)
    x = torch.from_numpy(rng.normal(0, 1.5, size=(2, 4, 2599)).astype(np.float32))
    for b, lab in enumerate(labels):
        for k in range(int(lens[b])):
            x[b, k, lab[k % len(lab)]] += 6.0
    call("ctc_v2599", "ctc", x, tgt, lens, tl, up=0.5)

    g["names"] = np.array(names)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(names)} calls")
    for n in names:
        gr = g[f"{n}__grad"]
        print(n, float(g[f"{n}__loss"]), "nan elements", int(np.isnan(gr).sum()), "non-zero", int((gr != 0).sum()))
    print("mp_ties grad:\n", g["mp_ties__grad"][..., 0], "\n", g["mp_ties__grad"][..., 1])
    print("mp_ties_dur2 grad col0:\n", g["mp_ties_dur2__grad"][..., 0])
    print("mp_clamp grad:\n", g["mp_clamp__grad"])
    print("ctc_infeasible NaN rows:\n", np.isnan(g["ctc_infeasible__grad"]).all(2).astype(int))
    print("ctc_infeasible NaN any:\n", np.isnan(g["ctc_infeasible__grad"]).any(2).astype(int))


if __name__ == "__main__":
    main()
