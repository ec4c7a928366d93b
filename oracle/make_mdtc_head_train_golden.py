#!/usr/bin/env python
"""Golden training-mode results of the speech-command MDTC model (test infrastructure): differentiates the REFERENCE's
own wekws/model/kws_model.py init_model MDTC with the `global` / `last` head in train() with torch's autograd on the
CPU, in float32 and in float64, as Executor.train does (logits -> loss -> loss.backward()), and writes
tests/golden/mdtc_head_train.npz.

The head's nn.Dropout (classifier.classifier.2) gets a forward hook that replaces its output by
input * where(mask, s, 0), the mask kws_mdtc_head_train_oracle.head_mask of the call's seed (s = 1.0f / (float)(1 - p)
in float32, 1 / (1 - p) in float64): this pins the documented mask function and the oracle to the reference model.
The seed is the one a training forward draws after torch.manual_seed(call_seed) (`call_seed`, `dseed`; 0 when p = 0,
where nothing is drawn); the mask is stored bit-packed (`mask`, np.packbits of the (B, 64) bools), with `p`.

Models: tests/head_cases.py HEAD_CASES with the weights build_head_model gives them (seed 777; pinned by
synth.state_digest as `digest_<case>`).  Per call <name>: the case, the features synth.features(B, T, idim, seed)
(`B`, `T`, `seed`, pinned by `feats_sum`), the float64 chain's upstream gradient (`up64`), the float32 and float64
logits (`logits`, `l64`) and the reference's float32-vs-float64 max error (`err32_l`); the float64 parameter gradients
and running statistics as kws_mdtc_train_oracle.digest fingerprints (`g64_digest`, `run64_digest`) and the reference's
own float32 error of each (`err32_g`, `err32_run`).  Calls:
  mdtc_global (examples/speechcommand_v1/s0/conf/mdtc.yaml: hidden 64, 80-dim MFCC, 11 outputs, global, p = 0.5)
    through the reference's `ce` loss, B = 4 one-second clips (T = 98);
  mdtc_last with a dense upstream gradient;
  mdtc_small_last (hidden 32, input 40) with a dense upstream gradient;
  mdtc_global with p = 0 and a dense upstream gradient.
      python oracle/make_mdtc_head_train_golden.py"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import kws_mdtc_head_train_oracle as KH  # noqa: E402
from oracle import kws_tcn_train_oracle as KT  # noqa: E402
from oracle.kws_mdtc_train_oracle import digest, running_names  # noqa: E402
from oracle.make_criterion_golden import import_reference  # noqa: E402
from tests.head_cases import build_head_model  # noqa: E402
from wekws_b200 import synth  # noqa: E402
from wekws_b200.frontend import draw_seed  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mdtc_head_train.npz")


def main():
    loss_mod, _ = import_reference()
    from wekws.model.kws_model import init_model
    rng = np.random.default_rng(2030)
    g, names, models = {}, [], {}
    for case in ("mdtc_global", "mdtc_last", "mdtc_small_last"):
        cfg, model = build_head_model(case, init_model)
        models[case] = (cfg, model)
        g[f"digest_{case}"] = np.float64(synth.state_digest(model))

    def chain(model0, cfg, feats, dtype, mask, p, loss):
        m = copy.deepcopy(model0).to(dtype)
        m.classifier.classifier[2].p = p
        m.train()
        s = KT.scale(p, dtype)
        mk = torch.from_numpy(mask)
        hook = m.classifier.classifier[2].register_forward_hook(
            lambda mod, inp, out: inp[0] * torch.where(mk, s, torch.zeros((), dtype=s.dtype)))
        logits, _ = m(feats.to(dtype))
        hook.remove()
        logits.retain_grad()
        loss(logits).backward()
        sd = m.state_dict()
        return (logits.detach().clone(), logits.grad.detach().clone(), [q.grad.detach().clone() for q in m.parameters()],
                [sd[k].detach().clone() for k in running_names(cfg["backbone"])], sd)

    def call(name, case, B, T, seed, call_seed, p=None, target=None):
        cfg, model = models[case]
        p = float(model.classifier.classifier[2].p) if p is None else p
        feats = synth.features(B, T, cfg["input_dim"], seed=seed)
        torch.manual_seed(call_seed)
        dseed = draw_seed() if p > 0 else 0
        mask = KH.head_mask(dseed, B, p)
        if target is not None:
            loss = lambda y: loss_mod.criterion("ce", y, target, torch.full((B,), T), None, 0, False)[0]
        else:
            up = torch.from_numpy(rng.normal(0, 1, size=(B, cfg["output_dim"])).astype(np.float32))
            loss = lambda y: (y * up.to(y.dtype)).sum()
        l32, _, g32, r32, sd32 = chain(model, cfg, feats, torch.float32, mask, p, loss)
        l64, up64, g64, r64, sd64 = chain(model, cfg, feats, torch.float64, mask, p, loss)
        for key in sd32:
            if key.endswith("num_batches_tracked"):
                assert int(sd32[key]) == int(sd64[key]) == int(model.state_dict()[key]) + 1
        rec = dict(case=np.array(case), B=np.int32(B), T=np.int32(T), seed=np.int64(seed), p=np.float64(p),
                   call_seed=np.int64(call_seed), dseed=np.uint64(dseed), mask=np.packbits(mask),
                   feats_sum=np.float64(feats.double().sum().item()), up64=up64.numpy(), logits=l32.numpy(),
                   l64=l64.numpy(), err32_l=np.float64((l32.double() - l64).abs().max().item()))
        for tag, a32, a64 in (("g", g32, g64), ("run", r32, r64)):
            rec[f"{tag}64_digest"] = torch.stack([digest(b) for b in a64]).numpy()
            rec[f"err32_{tag}"] = np.array([(a.double() - b).abs().max().item() for a, b in zip(a32, a64)])
        for k, v in rec.items():
            g[f"{name}__{k}"] = np.asarray(v)
        names.append(name)

    call("global_ce_T98", "mdtc_global", 4, 98, 801, 21, target=torch.from_numpy(rng.integers(0, 11, size=4)).long())
    call("last_dense_T40", "mdtc_last", 4, 40, 802, 22)
    call("small_last_dense_T30", "mdtc_small_last", 3, 30, 803, 23)
    call("global_p0_dense_T20", "mdtc_global", 3, 20, 804, 24, p=0.0)

    g["names"] = np.array(names)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(names)} calls")
    for n in names:
        print(n, "float32-vs-float64 max gradient error", float(g[f"{n}__err32_g"].max()), "logits", g[f"{n}__err32_l"])


if __name__ == "__main__":
    main()
