#!/usr/bin/env python
"""Golden training-mode results of the TCN / DS-TCN models (test infrastructure): differentiates the REFERENCE's own
wekws/model/kws_model.py init_model TCN / DS-TCN in train() with torch's autograd on the CPU, in float32 and in
float64, as Executor.train does (logits -> loss -> loss.backward()), and writes tests/golden/tcn_train.npz.

Every reference nn.Dropout gets a forward hook that replaces its output by input * where(mask, s, 0), the mask
kws_tcn_train_oracle.dropout_mask of the call's seed (s = 1.0f / (float)(1 - p) in float32, 1 / (1 - p) in float64):
this pins the documented mask function and the oracle to the reference model.  The seed is the one a training forward
draws after torch.manual_seed(call_seed) (`call_seed`, `seed`); the masks themselves are stored bit-packed (`masks`,
np.packbits of the (L, B, T, C) bools).

Models: kws_tcn_train_oracle.GOLDEN_CASES with the weights golden_model gives them (seed 777; pinned by
synth.state_digest as `digest_<case>`).  Per call <name>: the case, the features synth.features(B, T, idim, seed,
cmvn_like=<case has CMVN>) (`B`, `T`, `seed`, pinned by `feats_sum`), the frame lengths, the float64 chain's upstream
gradient (`up64`), the float32 and float64 logits (`logits`, `l64`) and the reference's float32-vs-float64 max error
(`err32_l`); the float64 parameter gradients and running statistics as kws_mdtc_train_oracle.digest fingerprints
(`g64_digest`, `run64_digest`) and the reference's own float32 error of each (`err32_g`, `err32_run`).  Calls:
  tcn (hidden 64) through the max-pooling loss on padded lengths;
  ds_tcn (hidden 256) with a dense upstream gradient;
  ds_tcn hidden 64 with global CMVN, dense upstream;
  ds_tcn_ctc (tests/cases.py: hidden 256, 37 tokens) through the reference's CTC loss on padded lengths;
  tcn with T = 5, shorter than the first block's padding of 7, dense upstream;
  ds_tcn hidden 64 with every p = 0, dense upstream.
      python oracle/make_tcn_train_golden.py"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import kws_tcn_train_oracle as KT  # noqa: E402
from oracle.kws_mdtc_train_oracle import digest  # noqa: E402
from oracle.make_criterion_golden import import_reference  # noqa: E402
from wekws_b200 import synth  # noqa: E402
from wekws_b200.frontend import draw_seed  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "tcn_train.npz")


def main():
    loss_mod, _ = import_reference()
    from wekws.model.kws_model import init_model
    rng = np.random.default_rng(2029)
    g, names, models = {}, [], {}
    for case in KT.GOLDEN_CASES:
        cfg, model = KT.golden_model(case, init_model)
        models[case] = (cfg, model)
        g[f"digest_{case}"] = np.float64(synth.state_digest(model))

    def chain(model0, cfg, feats, dtype, masks, ps, loss):
        m = copy.deepcopy(model0).to(dtype)
        m.train()
        hooks = []
        for l, d in enumerate(KT.block_dropouts(m)):
            s = KT.scale(ps[l], dtype)
            mk = torch.from_numpy(masks[l]).transpose(1, 2)                     # (B, C, T) as the block sees it
            hooks.append(d.register_forward_hook(
                lambda mod, inp, out, mk=mk, s=s: inp[0] * torch.where(mk, s, torch.zeros((), dtype=s.dtype))))
        logits, _ = m(feats.to(dtype))
        for h in hooks:
            h.remove()
        logits.retain_grad()
        loss(logits).backward()
        sd = m.state_dict()
        return (logits.detach().clone(), logits.grad.detach().clone(), [p.grad.detach().clone() for p in m.parameters()],
                [sd[k].detach().clone() for k in KT.running_names(cfg["backbone"])], sd)

    def call(name, case, B, T, seed, call_seed, kind="dense", lens=None, target=None, tlens=None):
        cfg, model = models[case]
        feats = synth.features(B, T, cfg["input_dim"], seed=seed, cmvn_like="cmvn" in cfg)
        ps = [d.p for d in KT.block_dropouts(model)]
        torch.manual_seed(call_seed)
        dseed = draw_seed()
        masks = KT.dropout_masks(dseed, B, T, cfg["hidden_dim"], ps)
        if kind == "dense":
            up = torch.from_numpy(rng.normal(0, 1, size=(B, T, cfg["output_dim"])).astype(np.float32))
            loss = lambda y: (y * up.to(y.dtype)).sum()
        elif kind == "max_pooling":
            loss = lambda y: loss_mod.criterion("max_pooling", y, target, lens, None, 0, False)[0]
        else:
            loss = lambda y: loss_mod.criterion("ctc", y, target, lens, tlens, 0, False)[0]
        l32, _, g32, r32, sd32 = chain(model, cfg, feats, torch.float32, masks, ps, loss)
        l64, up64, g64, r64, sd64 = chain(model, cfg, feats, torch.float64, masks, ps, loss)
        for key in sd32:
            if key.endswith("num_batches_tracked"):
                assert int(sd32[key]) == int(sd64[key]) == int(model.state_dict()[key]) + 1
        rec = dict(case=np.array(case), B=np.int32(B), T=np.int32(T), seed=np.int64(seed),
                   call_seed=np.int64(call_seed), dseed=np.uint64(dseed), masks=np.packbits(np.stack(masks)),
                   feats_sum=np.float64(feats.double().sum().item()), up64=up64.numpy(), logits=l32.numpy(),
                   l64=l64.numpy(), err32_l=np.float64((l32.double() - l64).abs().max().item()),
                   lens=(lens if lens is not None else torch.full((B,), T)).numpy())
        for tag, a32, a64 in (("g", g32, g64), ("run", r32, r64)):
            rec[f"{tag}64_digest"] = torch.stack([digest(b) for b in a64]).numpy()
            rec[f"err32_{tag}"] = np.array([(a.double() - b).abs().max().item() for a, b in zip(a32, a64)])
        for k, v in rec.items():
            g[f"{name}__{k}"] = np.asarray(v)
        names.append(name)

    B, T = 3, 40
    lens = torch.from_numpy(rng.integers(T // 2, T + 1, size=B)).long()
    lens[0] = T
    call("tcn_maxpool_T40", "tcn", B, T, 701, 11, "max_pooling", lens=lens, target=torch.zeros(B, dtype=torch.long))
    call("ds_tcn_dense_T30", "ds_tcn", 2, 30, 702, 12)
    call("ds_tcn64_cmvn_T50", "ds_tcn64_cmvn", 2, 50, 703, 13)
    B, T = 3, 50
    lens = torch.from_numpy(rng.integers(30, T + 1, size=B)).long()
    lens[0] = T
    tlens = torch.tensor([4, 3, 2])
    target = torch.from_numpy(rng.integers(1, 37, size=(B, 4))).long()
    call("ds_tcn_ctc_T50", "ds_tcn_ctc", B, T, 704, 14, "ctc", lens=lens, target=target, tlens=tlens)
    call("tcn_dense_T5", "tcn", 4, 5, 705, 15)
    call("ds_tcn64_p0_T20", "ds_tcn64_p0", 2, 20, 706, 16)

    g["names"] = np.array(names)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(names)} calls")
    for n in names:
        print(n, "float32-vs-float64 max gradient error", float(g[f"{n}__err32_g"].max()), "logits", g[f"{n}__err32_l"])


if __name__ == "__main__":
    main()
