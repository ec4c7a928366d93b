"""Generates tests/golden/config_sweep.npz from the REAL reference for a few rows of tests/test_config_sweep.py:

    python oracle/make_sweep_golden.py

For each of GOLDEN_ROWS it imports the reference's init_model read-only from /root/reference, gives the model the
project's synthetic weights (synth.randomize_, seed 777) and runs two calls: a 1 s clip from a random cache, then 9
frames with the cache carried.  Only outputs are stored, with the state-dict digest and the absolute sums of the inputs:
the tests rebuild the weights and inputs from their seeds and check them against these.  Keys are "<row>/<name>".
TEST INFRASTRUCTURE ONLY.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")

from wekws_b200 import synth                                                       # noqa: E402
from tests.test_config_sweep import GOLDEN_ROWS, build_row, golden_inputs          # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "config_sweep.npz")


def gen(row: str, arrays: dict) -> None:
    from wekws.model.kws_model import init_model
    cfg, model = build_row(row, init_model)
    x0, cache, x1 = golden_inputs(cfg)
    arrays[row + "/digest"] = np.float64(synth.state_digest(model))
    for name, t in (("x0", x0), ("cache", cache), ("x1", x1)):
        arrays[f"{row}/{name}_abs_sum"] = np.float64(t.double().abs().sum())
    with torch.no_grad():
        y0, c = model(x0, cache)
        y1, c = model(x1, c)
    arrays[row + "/y0"], arrays[row + "/y1"] = y0.numpy(), y1.numpy()
    arrays[row + "/c1_tail"] = c[..., -16:].contiguous().numpy()
    print(row, "y0", tuple(y0.shape), "y1", tuple(y1.shape), "cache", tuple(c.shape))


if __name__ == "__main__":
    arrays = {}
    for row in GOLDEN_ROWS:
        gen(row, arrays)
    np.savez_compressed(OUT, **arrays)
