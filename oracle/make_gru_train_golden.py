#!/usr/bin/env python
"""Golden training-mode results of the GRU model (test infrastructure): differentiates the REFERENCE's own
wekws/model/kws_model.py init_model GRU model in train() with torch's autograd on the CPU, in float32 and in float64,
as Executor.train does (logits -> loss -> loss.backward()), and writes tests/golden/gru_train.npz.

Models: kws_gru_train_oracle.GOLDEN_CASES with the weights golden_model gives them (seed 777; pinned by
synth.state_digest as `digest_<case>`).  Per call <name>: the case, the features synth.features(B, T, idim, seed,
cmvn_like=<case has CMVN>) (`B`, `T`, `seed`, pinned by `feats_sum`), the frame lengths, the float64 chain's upstream
gradient (`up64`), the float32 and float64 logits (`logits`, `l64`) and the reference's float32-vs-float64 max error
(`err32_l`); the float64 parameter gradients as kws_mdtc_train_oracle.digest fingerprints (`g64_digest`) and the
reference's own float32 error of each (`err32_g`).  Calls:
  gru (examples/hi_xiaowen/s0/conf/gru.yaml: input_dim 40, output_dim 2, global CMVN) through the max-pooling loss
    on padded lengths;
  gru_l1_i80 (1 layer, input_dim 80, output_dim 1, no CMVN) with a dense upstream gradient;
  gru_l4_id37 (4 layers, Identity, output_dim 37) with a dense upstream gradient;
  gru with T = 1 and B = 1, dense upstream.
      python oracle/make_gru_train_golden.py"""
import copy
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import kws_gru_train_oracle as KG  # noqa: E402
from oracle.kws_mdtc_train_oracle import digest  # noqa: E402
from oracle.make_criterion_golden import import_reference  # noqa: E402
from wekws_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "gru_train.npz")


def main():
    loss_mod, _ = import_reference()
    from wekws.model.kws_model import init_model
    rng = np.random.default_rng(2031)
    g, names, models = {}, [], {}
    for case in KG.GOLDEN_CASES:
        cfg, model = KG.golden_model(case, init_model)
        assert [n for n, _ in model.named_parameters()] == KG.param_names(cfg["backbone"]["num_layers"])
        models[case] = (cfg, model)
        g[f"digest_{case}"] = np.float64(synth.state_digest(model))

    def chain(model0, feats, dtype, loss):
        m = copy.deepcopy(model0).to(dtype)
        m.train()
        # the reference's GRU refuses its default empty cache: start of stream is an explicit zero state
        h0 = torch.zeros(m.backbone.num_layers, feats.shape[0], m.backbone.hidden_size, dtype=dtype)
        logits, _ = m(feats.to(dtype), h0)
        logits.retain_grad()
        loss(logits).backward()
        return logits.detach().clone(), logits.grad.detach().clone(), [p.grad.detach().clone() for p in m.parameters()]

    def call(name, case, B, T, seed, kind="dense", lens=None, target=None):
        cfg, model = models[case]
        feats = synth.features(B, T, cfg["input_dim"], seed=seed, cmvn_like="cmvn" in cfg)
        if kind == "dense":
            up = torch.from_numpy(rng.normal(0, 1, size=(B, T, cfg["output_dim"])).astype(np.float32))
            loss = lambda y: (y * up.to(y.dtype)).sum()
        else:
            loss = lambda y: loss_mod.criterion("max_pooling", y, target, lens, None, 0, False)[0]
        l32, _, g32 = chain(model, feats, torch.float32, loss)
        l64, up64, g64 = chain(model, feats, torch.float64, loss)
        rec = dict(case=np.array(case), B=np.int32(B), T=np.int32(T), seed=np.int64(seed),
                   feats_sum=np.float64(feats.double().sum().item()), up64=up64.numpy(), logits=l32.numpy(),
                   l64=l64.numpy(), err32_l=np.float64((l32.double() - l64).abs().max().item()),
                   lens=(lens if lens is not None else torch.full((B,), T)).numpy(),
                   g64_digest=torch.stack([digest(b) for b in g64]).numpy(),
                   err32_g=np.array([(a.double() - b).abs().max().item() for a, b in zip(g32, g64)]))
        for k, v in rec.items():
            g[f"{name}__{k}"] = np.asarray(v)
        names.append(name)

    B, T = 3, 60
    lens = torch.from_numpy(rng.integers(T // 2, T + 1, size=B)).long()
    lens[0] = T
    call("gru_maxpool_T60", "gru", B, T, 801, "max_pooling", lens=lens, target=torch.tensor([0, 1, -1]))
    call("gru_l1_i80_dense_T40", "gru_l1_i80", 2, 40, 802)
    call("gru_l4_id37_dense_T25", "gru_l4_id37", 2, 25, 803)
    call("gru_dense_T1_B1", "gru", 1, 1, 804)

    g["names"] = np.array(names)
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(names)} calls")
    for n in names:
        print(n, "float32-vs-float64 max gradient error", float(g[f"{n}__err32_g"].max()), "logits", g[f"{n}__err32_l"])


if __name__ == "__main__":
    main()
