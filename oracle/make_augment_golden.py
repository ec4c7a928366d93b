"""Writes tests/golden/augment.npz from the reference itself (run with the reference checkout on sys.path):

* ``rv``: wekws/dataset/processor.py add_reverb on each row of the seeded batch (kws_augment_oracle.audio, at the
  reference's [-1, 1] scale) with a stub source serving kws_augment_oracle.rir_items (RIRs of 1, 31, 4000 and 16000
  taps, int16 and float32 WAVs, a stereo file), under a seeded ``random``;
* ``nz``: add_noise likewise with kws_augment_oracle.noise_items (all four key prefixes; clips shorter than, equal to
  and longer than the rows);
* ``snips`` / ``snips_sa``: the hey_snips ds_tcn dataset_conf chain (reverb_prob 0.2, noise_prob 0.3, fbank 40 with
  dither 1.0), utterance by utterance as Dataset() runs it: add_reverb, add_noise, compute_fbank with torch.randn
  patched to the restated dither noise (as oracle/make_train_features_golden.py does), [spec_aug], padding().
  ``snips_sa`` turns spec_aug on with the config's spec_aug_conf, to pin the interleaving of the draws.

Each case's seed is the first that exercises everything the case is for (every clip or prefix, rows selected and
skipped).  The stub source draws its key as LmdbData.random_one does.  Every ``random`` call is logged
(kws_augment_oracle.Recorder) and stored as JSON; the outputs are stored as the reference returns them (for the
stage cases, only the rows it changed, one after the other).  Inputs are
not stored: they come from seeds.

    python oracle/make_augment_golden.py [/path/to/reference]
"""
import json
import os
import sys
from unittest import mock

import numpy as np
import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = sys.argv[1] if len(sys.argv) > 1 else "/root/reference"
sys.path.insert(0, REF)

from oracle import kws_augment_oracle as A  # noqa: E402
from oracle import kws_train_oracle as T  # noqa: E402
from wekws.dataset import processor  # noqa: E402

GEN_SEED = 4321


class StubSource:
    """keys + random_one() over (key, bytes) items, drawing the index as LmdbData.random_one does."""

    def __init__(self, items, rnd):
        self.keys = [k for k, _ in items]
        self.data = dict(items)
        self.rnd = rnd

    def random_one(self):
        key = self.keys[self.rnd.randint(0, len(self.keys) - 1)]
        return key, self.data[key]


def draw_seed(gen_seed):
    lo, hi = torch.randint(0, 1 << 32, (2,), dtype=torch.int64, generator=torch.Generator().manual_seed(gen_seed)).tolist()
    return lo | (hi << 32)


def stage_case(kind, items, prob, want):
    pcm, lens = A.audio()
    fn = processor.add_reverb if kind == "reverb" else processor.add_noise
    for seed in range(1000):
        rec = A.Recorder(seed)
        src = StubSource(items, rec)
        out = []
        with mock.patch.object(processor, "random", rec):
            for b, n in enumerate(lens):
                s = {"key": f"utt{b}", "wav": torch.from_numpy(pcm[b:b + 1, :n].astype(np.float32) / (1 << 15))}
                out.append(next(fn(iter([s]), src, prob))["wav"].numpy()[0])
        picks = A.replay(rec.dumps(), lens, items, kind)
        if want(picks, lens):      # only the selected rows are stored, one after the other
            return seed, np.concatenate([y for y, p in zip(out, picks) if p is not None]), rec.dumps()
    raise RuntimeError(f"no seed covers the {kind} case")


def reverb_covered(picks, lens):
    used = {p for p in picks if p is not None}
    return len(used) == len(A.rir_items()) and None in picks


def noise_covered(picks, lens):
    items = A.noise_items()
    sel = [(b, p) for b, p in enumerate(picks) if p is not None]
    prefixes = {items[p[0]][0].split("_")[0] for _, p in sel}
    clip_len = [len(A.decode(v)) for _, v in items]
    rel = {np.sign(clip_len[p[0]] - lens[b]) for b, p in sel}
    return prefixes == {"noise", "speech", "music", "babble"} and rel == {-1, 0, 1} and None in picks


def chain(name, conf, out, spec_aug):
    pcm, lens = A.audio()
    B = len(lens)
    keys = [f"{name}_utt{b}" for b in range(B)]
    labels = [int(v) for v in np.random.default_rng(24).integers(-1, 4, B)]
    seed = draw_seed(GEN_SEED)
    noise = torch.from_numpy(T.dither_noise(seed, B, max(T.O.num_frames(n) for n in lens))).float()
    conf = dict(conf, spec_aug=spec_aug)
    rv_items, nz_items = A.rir_items(), A.noise_items()

    def run(rng_seed):
        rec = A.Recorder(rng_seed)
        rv, nz = StubSource(rv_items, rec), StubSource(nz_items, rec)
        samples, events = [], []
        with mock.patch.object(processor, "random", rec):
            for b in range(B):
                s = {"key": keys[b], "label": labels[b], "sample_rate": 16000,
                     "wav": torch.from_numpy(pcm[b:b + 1, :lens[b]].astype(np.float32) / (1 << 15))}
                w0 = s["wav"]
                s = next(processor.add_reverb(iter([s]), rv, conf["reverb_prob"]))
                w1 = s["wav"]
                s = next(processor.add_noise(iter([s]), nz, conf["noise_prob"]))
                events.append([w1 is not w0, s["wav"] is not w1])
                m = T.O.num_frames(lens[b])
                with mock.patch.object(torch, "randn", lambda *a, _n=noise[b, :m], **k: _n.clone()):
                    s = next(processor.compute_fbank(iter([s]), **conf["fbank_conf"]))
                if spec_aug:
                    s = next(processor.spec_aug(iter([s]), **conf.get("spec_aug_conf", {})))
                samples.append(s)
        return next(processor.padding(iter([samples]))), rec.dumps(), events

    for rng_seed in range(1000):
        res, log, events = run(rng_seed)
        if sum(e[0] for e in events) >= 2 and sum(e[1] for e in events) >= 2:
            break
    k, feats, target, flens, tlens = res
    p = name + "_"
    out.update({p + "keys": np.array(keys), p + "labels": json.dumps(labels), p + "conf": json.dumps(conf),
                p + "seed": np.uint64(seed), p + "rng_seed": rng_seed, p + "log": log,
                p + "events": np.array(events), p + "out_keys": np.array(k), p + "feats": feats.numpy(),
                p + "target": target.numpy(), p + "feats_lengths": flens.numpy(), p + "target_lengths": tlens.numpy()})


def main():
    out = {"gen_seed": GEN_SEED}
    seed, y, log = stage_case("reverb", A.rir_items(), 0.75, reverb_covered)
    out.update(rv_seed=seed, rv_prob=0.75, rv_out=y, rv_log=log)
    seed, y, log = stage_case("noise", A.noise_items(), 0.75, noise_covered)
    out.update(nz_seed=seed, nz_prob=0.75, nz_out=y, nz_log=log)
    conf = yaml.safe_load(open(os.path.join(REF, "examples/hey_snips/s0/conf/ds_tcn.yaml")))["dataset_conf"]
    chain("snips", conf, out, spec_aug=False)
    chain("snips_sa", conf, out, spec_aug=True)
    path = os.path.join(ROOT, "tests", "golden", "augment.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes; seeds", out["rv_seed"], out["nz_seed"],
          out["snips_rng_seed"], out["snips_sa_rng_seed"])


if __name__ == "__main__":
    main()
