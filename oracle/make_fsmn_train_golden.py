#!/usr/bin/env python
"""Golden parameter gradients of the FSMN model (test infrastructure): differentiates the REFERENCE's own
wekws/model/kws_model.py init_model FSMN in training mode with torch's autograd on the CPU, in float32 and in float64,
as Executor.train does (logits -> loss.py criterion -> loss.backward()), and writes tests/golden/fsmn_train.npz.

Models: both FSMN_CASES configs of tests/cases.py, each with global CMVN (norm_var true) and with mean-only CMVN
(norm_var false).  Per config <case>: the state_dict both its models share (`sd_<case>__<key>`) and the parameter
names in state_dict order (`names_<case>`).  Per model `m<k>`: its case and norm_var.  Per call <name>: the model,
the features as synth.features(B, T, 40, seed, cmvn_like=True) (`B`, `T`, `seed` and the float64 sum `feats_sum`
that pins them), the frame lengths, the upstream gradient d loss / d logits of the float64 chain (`up64`; the float32
chain's is its rounding for the dense upstream, and its own CTC gradient otherwise), the float32 logits, each parameter's float64 gradient (`g64_<i>`, i in
state_dict order) and the reference's own float32-vs-float64 error of it (`err32_<i>`, max abs).  Four calls, one per
model, together cover: T = 5 (thirteen streams share a 64-row tile), 64 (one stream fills a tile) and 150 (three
time chunks), padded lengths with the loss of the reference's CTC criterion on them (padding rows get exact zeros),
and an upstream gradient that is random on every row.
      python oracle/make_fsmn_train_golden.py"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.make_criterion_golden import import_reference, padded  # noqa: E402
from tests.cases import FSMN_CASES, fsmn_config  # noqa: E402
from wekws_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "fsmn_train.npz")


def param_names(model):
    return [n for n, _ in model.named_parameters()]


def main():
    loss_mod, _ = import_reference()
    from wekws.model.kws_model import init_model
    rng = np.random.default_rng(2027)
    g, names, models = {}, [], []

    def chain(model, feats, dtype, lens=None, labels=None, up=None):
        m = model.to(dtype)
        m.train()
        m.zero_grad(set_to_none=True)
        logits, _ = m(feats.to(dtype))
        logits.retain_grad()
        if up is None:
            tgt, tl = padded(labels)
            loss, _ = loss_mod.criterion("ctc", logits, tgt, lens, tl, 0, False)
        else:
            loss = (logits * up.to(dtype)).sum()
        loss.backward()
        return logits.detach().clone(), logits.grad.detach().clone(), [p.grad.detach().clone()
                                                                       for p in m.parameters()]

    def call(name, mk, model, B, T, seed, lens=None, labels=None, up=None):
        feats = synth.features(B, T, 40, seed=seed, cmvn_like=True)
        l32, _, g32 = chain(model, feats, torch.float32, lens, labels, up)
        _, up64, g64 = chain(model, feats, torch.float64, lens, labels, up)
        model.float()
        rec = dict(model=np.int32(mk), B=np.int32(B), T=np.int32(T), seed=np.int64(seed),
                   feats_sum=np.float64(feats.double().sum().item()), up64=up64, logits=l32)
        rec["lens"] = lens if lens is not None else torch.full((B,), T)
        for i, (a, b) in enumerate(zip(g32, g64)):
            rec[f"g64_{i}"] = b
            rec[f"err32_{i}"] = np.float64((a.double() - b).abs().max().item())
        for k, v in rec.items():
            g[f"{name}__{k}"] = v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        names.append(name)

    V = 7
    for case in FSMN_CASES:
        for norm_var in (True, False):
            cfg = fsmn_config(case)
            cmvn_file = synth.write_cmvn_json(cfg["input_dim"], seed=11)
            try:
                cfg["cmvn"] = dict(cmvn_file=cmvn_file, norm_var=norm_var)
                with contextlib.redirect_stdout(io.StringIO()):
                    torch.manual_seed(777)
                    model = init_model(cfg)
            finally:
                os.unlink(cmvn_file)
            mk = len(models)
            models.append((case, norm_var))
            for k, v in model.state_dict().items():             # the same for both norm_var settings
                if f"sd_{case}__{k}" in g:
                    assert np.array_equal(g[f"sd_{case}__{k}"], v.numpy())
                g[f"sd_{case}__{k}"] = v.numpy()
            g[f"names_{case}"] = np.array(param_names(model))
            g[f"m{mk}__case"], g[f"m{mk}__norm_var"] = np.array(case), np.int32(norm_var)
            if mk < 3:                                         # CTC on padded lengths, T below / at / above a tile
                T, B = ((5, 13), (64, 2), (150, 2))[mk]
                lens = torch.from_numpy(rng.integers(max(3, T // 2), T + 1, size=B)).long()
                lens[0] = T
                labels = [list(rng.choice(np.arange(1, V), size=int(rng.integers(1, 3)), replace=False))
                          for _ in range(B)]
                call(f"m{mk}_ctc_T{T}", mk, model, B, T, 500 + 10 * mk + T, lens=lens, labels=labels)
            else:                                              # a dense upstream gradient: every row exercised
                up = torch.from_numpy(rng.normal(0, 1, size=(3, 64, V)).astype(np.float32))
                call(f"m{mk}_dense_T64", mk, model, 3, 64, 900 + mk, up=up)

    g["names"] = np.array(names)
    g["num_models"] = np.int32(len(models))
    np.savez_compressed(OUT, **g)
    print(f"wrote {OUT}: {os.path.getsize(OUT)} bytes, {len(names)} calls")
    for n in names:
        count = len([key for key in g if key.startswith(f"{n}__err32_")])
        err = max(float(g[f"{n}__err32_{i}"]) for i in range(count))
        print(n, "logits", g[f"{n}__logits"].shape, "float32-vs-float64 max gradient error", err)


if __name__ == "__main__":
    main()
