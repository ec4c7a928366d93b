"""Writes tests/golden/train_features.npz from the reference itself (run with the reference checkout on sys.path):

* ``spec_aug``: wekws/dataset/processor.py spec_aug on each row of a ragged batch under a seeded ``random`` state
  (defaults 2 / 2 / 50 / 10, rows shorter than max_t, masks that run past the end);
* three training chains, the ds_tcn (fbank 40), mdtc (legacy mfcc 80) and fsmn_ctc (fbank 80, context 2 / 2,
  frame_skip 3) dataset_conf of examples/hi_xiaowen/s0/conf: compute_fbank / compute_mfcc with their dither 1.0 and
  torch.randn patched to return the restated dither noise (oracle/kws_train_oracle.py) of the row, spec_aug under a
  seeded ``random``, context_expansion, frame_skip and padding(), utterance by utterance as Dataset() runs them.

The inputs are not stored: they come from seeds (kws_train_oracle.golden_audio / spec_aug_input).  The spec_aug
result is stored as the packed bit mask of its zeros (every other element is the input).  The dither seed is the one
wekws_b200.TrainFeatures draws from torch.Generator().manual_seed(GEN_SEED): two 32-bit torch.randint draws, low word
first.

    python oracle/make_train_features_golden.py [/path/to/reference]
"""
import json
import os
import random
import sys
from unittest import mock

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
sys.path.insert(0, REF)

from oracle import kws_train_oracle as T  # noqa: E402
from wekws.dataset import processor  # noqa: E402

CONFIGS = {"ds_tcn": "ds_tcn.yaml", "mdtc": "mdtc.yaml", "fsmn_ctc": "fsmn_ctc.yaml"}
GEN_SEED, RNG_SEED = 1234, 99


def draw_seed(gen_seed):
    lo, hi = torch.randint(0, 1 << 32, (2,), dtype=torch.int64, generator=torch.Generator().manual_seed(gen_seed)).tolist()
    return lo | (hi << 32)


def spec_aug_case(out):
    x, frames = T.spec_aug_input()
    assert not (x == 0).any()
    expect = x.copy()
    random.seed(7)
    for b, n in enumerate(frames):
        y = next(processor.spec_aug(iter([{"feat": torch.from_numpy(x[b, :n].copy())}])))["feat"]
        expect[b, :n] = y.numpy()
    assert np.array_equal(expect[expect != 0], x[expect != 0])
    out.update(sa_zero=np.packbits(expect == 0), sa_rng_seed=7)


def chain(name, conf, out):
    pcm, lens = T.golden_audio()
    B = len(lens)
    rng = np.random.default_rng(12)
    keys = [f"{name}_utt{b}" for b in range(B)]
    if name == "fsmn_ctc":
        labels = [[int(v) for v in rng.integers(1, 2599, int(rng.integers(1, 6)))] for _ in range(B)]
    else:
        labels = [int(v) for v in rng.integers(-1, 2, B)]
    seed = draw_seed(GEN_SEED)
    noise = torch.from_numpy(T.dither_noise(seed, B, max(T.O.num_frames(n) for n in lens))).float()
    if "feats_type" in conf:
        feat_conf, fn = dict(conf["fbank_conf"]), processor.compute_fbank
    else:
        feat_conf = dict(conf["feature_extraction_conf"])
        fn = processor.compute_mfcc if feat_conf["feature_type"] == "mfcc" else processor.compute_fbank

    def run():
        random.seed(RNG_SEED)
        samples = []
        for b in range(B):
            s = {"key": keys[b], "label": labels[b], "sample_rate": 16000,
                 "wav": torch.from_numpy(pcm[b:b + 1, :lens[b]].astype(np.float32) / (1 << 15))}
            m = T.O.num_frames(lens[b])
            with mock.patch.object(torch, "randn", lambda *a, _n=noise[b, :m], **k: _n.clone()):
                s = next(fn(iter([s]), **feat_conf))
            if conf.get("spec_aug", True):
                s = next(processor.spec_aug(iter([s]), **conf.get("spec_aug_conf", {})))
            if conf.get("context_expansion", False):
                s = next(processor.context_expansion(iter([s]), **conf.get("context_expansion_conf", {})))
            if conf.get("frame_skip", 1) > 1:
                s = next(processor.frame_skip(iter([s]), conf["frame_skip"]))
            samples.append(s)
        return next(processor.padding(iter([samples])))

    k, feats, target, flens, tlens = run()
    p = name + "_"
    out.update({p + "keys": np.array(keys),
                p + "labels": json.dumps(labels), p + "conf": json.dumps(conf), p + "seed": np.uint64(seed),
                p + "out_keys": np.array(k), p + "feats": feats.numpy(), p + "target": target.numpy(),
                p + "feats_lengths": flens.numpy(), p + "target_lengths": tlens.numpy()})


def main():
    out = {"gen_seed": GEN_SEED, "rng_seed": RNG_SEED}
    spec_aug_case(out)
    for name, f in CONFIGS.items():
        conf = yaml.safe_load(open(os.path.join(REF, "examples/hi_xiaowen/s0/conf", f)))["dataset_conf"]
        chain(name, conf, out)
    path = os.path.join(ROOT, "tests", "golden", "train_features.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
