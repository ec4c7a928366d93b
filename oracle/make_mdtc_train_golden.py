#!/usr/bin/env python
"""Golden training-mode results of the MDTC model (test infrastructure): differentiates the REFERENCE's own
wekws/model/kws_model.py init_model MDTC in training mode with torch's autograd on the CPU, in float32 and in float64,
as Executor.train does (logits -> loss -> loss.backward()), and writes tests/golden/mdtc_train.npz.

Models: the three MDTC cases of tests/cases.py (mdtc: hidden 64, 17 blocks; mdtc_small: hidden 32, input 40;
mdtc_cmvn_logits: global CMVN, identity activation, output 2), with the weights tests.cases.build_model gives them
(seed 777; not stored, pinned by synth.state_digest as `digest_<case>`).  Per call <name>: the case, the features as
synth.features(B, T, idim, seed, cmvn_like=<case has CMVN>) (`B`, `T`, `seed` and the float64 sum `feats_sum` that pins
them), the frame lengths, the upstream gradient d loss / d logits of the float64 chain (`up64`), the float32 logits
and the float64 logits (`l64`) with the reference's own float32-vs-float64 max abs error of the logits (`err32_l`).
For the parameter gradients (named_parameters order) and the BatchNorm running statistics after the call
(kws_mdtc_train_oracle.running_names order): the float64 values as kws_mdtc_train_oracle.digest fingerprints, one row
per tensor (`g64_digest`, `run64_digest`; the full tensors of the hidden-64 models would take megabytes), and the
reference's own float32-vs-float64 max abs error of each tensor (`err32_g`, `err32_run`).  Calls:
  T = 5, shorter than the padding of every dilated block (tiny B * T statistics), dense upstream (mdtc_small);
  padded lengths through the reference's max-pooling loss, keyword targets (mdtc, mdtc_small);
  T = 150 with a dense upstream (mdtc_cmvn_logits).
      python oracle/make_mdtc_train_golden.py"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.kws_mdtc_train_oracle import digest, running_names  # noqa: E402
from oracle.make_criterion_golden import import_reference  # noqa: E402
from tests.cases import build_model  # noqa: E402
from wekws_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mdtc_train.npz")


def main():
    loss_mod, _ = import_reference()
    from wekws.model.kws_model import init_model
    rng = np.random.default_rng(2028)
    g, names = {}, []
    models = {}
    for case in ("mdtc", "mdtc_small", "mdtc_cmvn_logits"):
        cfg, model, _ = build_model(case, init_model)
        models[case] = (cfg, model)
        g[f"digest_{case}"] = np.float64(synth.state_digest(model))

    def chain(model0, cfg, feats, dtype, lens, target, up):
        m = copy.deepcopy(model0).to(dtype)
        m.train()
        logits, _ = m(feats.to(dtype))
        logits.retain_grad()
        if up is None:
            loss, _ = loss_mod.criterion("max_pooling", logits, target, lens, None, 0, False)
        else:
            loss = (logits * up.to(dtype)).sum()
        loss.backward()
        sd = m.state_dict()
        return (logits.detach().clone(), logits.grad.detach().clone(), [p.grad.detach().clone() for p in m.parameters()],
                [sd[k].detach().clone() for k in running_names(cfg["backbone"])], sd)

    def call(name, case, B, T, seed, lens=None, target=None, dense=False):
        cfg, model = models[case]
        feats = synth.features(B, T, cfg["input_dim"], seed=seed, cmvn_like="cmvn" in cfg)
        up = torch.from_numpy(rng.normal(0, 1, size=(B, T, cfg["output_dim"])).astype(np.float32)) if dense else None
        l32, _, g32, r32, sd32 = chain(model, cfg, feats, torch.float32, lens, target, up)
        l64, up64, g64, r64, sd64 = chain(model, cfg, feats, torch.float64, lens, target, up)
        for key in sd32:
            if key.endswith("num_batches_tracked"):
                assert int(sd32[key]) == int(sd64[key]) == int(model.state_dict()[key]) + 1
        rec = dict(case=np.array(case), B=np.int32(B), T=np.int32(T), seed=np.int64(seed),
                   feats_sum=np.float64(feats.double().sum().item()), up64=up64.numpy(), logits=l32.numpy(),
                   l64=l64.numpy(), err32_l=np.float64((l32.double() - l64).abs().max().item()),
                   lens=(lens if lens is not None else torch.full((B,), T)).numpy())
        for tag, a32, a64 in (("g", g32, g64), ("run", r32, r64)):
            rec[f"{tag}64_digest"] = torch.stack([digest(b) for b in a64]).numpy()
            rec[f"err32_{tag}"] = np.array([(a.double() - b).abs().max().item() for a, b in zip(a32, a64)])
        for k, v in rec.items():
            g[f"{name}__{k}"] = np.asarray(v)
        names.append(name)

    call("small_dense_T5", "mdtc_small", 3, 5, 601, dense=True)
    for case, B, T, seed in (("mdtc", 4, 40, 602), ("mdtc_small", 3, 64, 603)):
        lens = torch.from_numpy(rng.integers(T // 2, T + 1, size=B)).long()
        lens[0] = T
        # keyword targets only: at these weights every utterance's max posterior is within 1e-3 of 1, where a
        # non-keyword utterance's -log(1 - p) amplifies the float32 rounding of 1 - p a thousandfold
        target = torch.zeros(B, dtype=torch.long)
        call(f"{case}_maxpool_T{T}", case, B, T, seed, lens=lens, target=target)
    call("cmvn_logits_dense_T150", "mdtc_cmvn_logits", 2, 150, 604, dense=True)

    g["names"] = np.array(names)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(names)} calls")
    for n in names:
        print(n, "logits", g[f"{n}__logits"].shape, "float32-vs-float64 max gradient error",
              float(g[f"{n}__err32_g"].max()))


if __name__ == "__main__":
    main()
