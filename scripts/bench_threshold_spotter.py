"""Per-call cost of the online threshold detector (wekws_b200.ThresholdSpotter) against the host loop a user writes
without it, for two max-pooling recipes of examples/hi_xiaowen: DS-TCN (40 mel, hidden 256) and MDTC (80 mel), both
with two keywords, synthetic weights, at several stream counts and chunk lengths.

Both sides run the same front half (StreamFrontEnd: PCM remainder, Fbank, the model with its cache) on their own
streams.  The spotter then detects on the device and copies its events back; the baseline copies the (frames, 2)
posteriors back with ``.cpu()`` and scans them in numpy with the same rule (compute_det.py:91-97, carried across
chunks).  The two alternate call by call in the same run.  Each call is timed with the host clock; both calls end in a
device-to-host copy, which synchronises.  Reported per model, B and chunk: p50 / p90 call time of each side and
streams served in real time (B * chunk / p50).  The card's name and power limit are read in the same run.  Prints one
JSON line.

    python scripts/bench_threshold_spotter.py [--batches 1024,4096] [--chunks-ms 100,500] [--calls 50] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from wekws_b200 import Fbank, ThresholdSpotter, init_model, model_config, synth      # noqa: E402
from wekws_b200.spotter import StreamFrontEnd                                         # noqa: E402

THRESHOLDS = [0.5, 0.5]
WINDOW_SHIFT = 50
MODELS = {"ds_tcn": 40, "mdtc": 80}             # recipe -> mel bins


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


class HostScan:
    """The baseline: the same front half and model, the posteriors copied to the host, the rule in numpy."""

    def __init__(self, model, B, fb):
        self.front = StreamFrontEnd(model, B, fb, 0, 0, 1, "baseline")
        K = model.odim
        self.thr = np.asarray(THRESHOLDS[:K], np.float64)
        self.seen = np.zeros((B, K), np.int64)
        self.next = np.zeros((B, K), np.int64)

    def __call__(self, pcm):
        c = self.front(pcm, None, 0)
        if c.probs is None:
            return []
        r6 = np.rint(c.probs.cpu().numpy().astype(np.float64) * 1e6) / 1e6
        T = int(c.nout[0])                      # every stream has the same frame count (one group)
        p = r6.reshape(-1, T, r6.shape[1])
        events = []
        for i in range(T):
            t = self.seen + i
            fire = (t >= self.next) & (p[:, i, :] >= self.thr)
            self.next = np.where(fire, t + WINDOW_SHIFT, self.next)
            b, k = np.nonzero(fire)
            events.append((b, k, t[b, k]))
        self.seen += T
        return events


def measure(name: str, B: int, chunk: int, calls: int, warmup: int, dev: str) -> dict:
    mel = MODELS[name]
    torch.manual_seed(777)
    model = synth.randomize_(init_model(model_config(name, input_dim=mel, output_dim=2))).eval().to(dev)
    fb = Fbank(mel)
    spot = ThresholdSpotter(model, THRESHOLDS, B, frontend=fb, window_shift=WINDOW_SHIFT)
    base = HostScan(model, B, fb)
    n = 8
    audio = synth.pcm_int16(B, chunk * n, seed=B).to(dev)
    chunks = [audio[:, i * chunk:(i + 1) * chunk] for i in range(n)]
    for i in range(warmup):
        spot(chunks[i % n])
        base(chunks[i % n])
    torch.cuda.synchronize()
    t_spot, t_base, fired = [], [], 0
    for i in range(calls):
        t0 = time.perf_counter()
        res = spot(chunks[i % n])
        t_spot.append(time.perf_counter() - t0)
        fired += int(res.counts.sum())
        t0 = time.perf_counter()
        base(chunks[i % n])
        t_base.append(time.perf_counter() - t0)
    out = {"model": name, "streams": B, "chunk_ms": chunk * 1000 // 16000, "calls": calls, "firings": fired}
    for side, t in (("spotter", t_spot), ("host_scan", t_base)):
        p50, p90 = float(np.percentile(t, 50)), float(np.percentile(t, 90))
        out[side] = {"p50_ms": p50 * 1e3, "p90_ms": p90 * 1e3, "realtime_streams": B * chunk / 16000 / p50}
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1024,4096")
    ap.add_argument("--chunks-ms", default="100,500")
    ap.add_argument("--models", default="ds_tcn,mdtc")
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_threshold_spotter.py needs a CUDA device")
    if args.calls < 10:
        raise SystemExit("--calls must be >= 10 for a p90")
    dev = "cuda:0"
    rows = [measure(name, int(B), int(ms) * 16, args.calls, args.warmup, dev) for name in args.models.split(",")
            for B in args.batches.split(",") for ms in args.chunks_ms.split(",")]
    print(json.dumps({"bench": "threshold_spotter", "window_shift": WINDOW_SHIFT, "card": card(), "results": rows}))


if __name__ == "__main__":
    main()
