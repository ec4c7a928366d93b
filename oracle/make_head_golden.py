"""Generates tests/golden/model_<case>.npz for the utterance-level classifier heads from the REAL reference:

    python oracle/make_head_golden.py

It imports the reference's init_model read-only from /root/reference, gives the model the project's synthetic weights
(synth.randomize_, seed 777) and stores the state-dict digest, keys and shapes, three chunks streamed with the cache
carried, one whole-utterance call of FULL_T frames and a batch of BATCH_B one-second clips.  The GPU box has no reference
checkout: the tests there compare against these files.  TEST INFRASTRUCTURE ONLY.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")

from wekws_b200 import synth                                                       # noqa: E402
from tests.head_cases import (BATCH_B, BATCH_SEED, BATCH_T, FULL_SEED, FULL_T, HEAD_B, HEAD_CASES,  # noqa: E402
                              HEAD_CHUNKS, build_head_model)

OUT = os.path.join(ROOT, "tests", "golden")


def gen(case: str) -> None:
    from wekws.model.kws_model import init_model
    cfg, model = build_head_model(case, init_model)
    idim = cfg["input_dim"]
    arrays = {"digest": np.float64(synth.state_digest(model)), "keys": np.array(sorted(model.state_dict().keys())),
              "shapes": np.array([list(model.state_dict()[k].shape) + [0] * (3 - model.state_dict()[k].dim())
                                  for k in sorted(model.state_dict().keys())], dtype=np.int64)}
    with torch.no_grad():
        cache = torch.zeros(0, 0, 0)
        for i, T in enumerate(HEAD_CHUNKS):
            x = synth.features(HEAD_B, T, idim, seed=500 + i)
            y, cache = model(x, cache)
            arrays[f"x{i}"], arrays[f"y{i}"] = x.numpy(), y.numpy()
        arrays[f"c{len(HEAD_CHUNKS) - 1}"] = cache.numpy()
        # the two long inputs are regenerated from their seeds by the tests (synth.features); the stored sums catch a
        # generator that draws differently
        x = synth.features(HEAD_B, FULL_T, idim, seed=FULL_SEED)
        y, c = model(x, torch.zeros(0, 0, 0))
        arrays["x_full_abs_sum"], arrays["y_full"], arrays["c_full"] = np.float64(x.double().abs().sum()), y.numpy(), c.numpy()
        x = synth.features(BATCH_B, BATCH_T, idim, seed=BATCH_SEED)
        y, _ = model(x, torch.zeros(0, 0, 0))
        arrays["x_batch_abs_sum"], arrays["y_batch"] = np.float64(x.double().abs().sum()), y.numpy()
    np.savez_compressed(os.path.join(OUT, f"model_{case}.npz"), **arrays)
    print(case, "keys", len(arrays["keys"]), "y_full", arrays["y_full"].shape)


if __name__ == "__main__":
    for case in HEAD_CASES:
        gen(case)
