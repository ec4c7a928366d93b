"""Per-call cost of the streaming keyword spotter (wekws_b200.KeywordSpotter): B live streams, one 0.3 s int16 chunk
per stream per call, for the two CTC recipes -- FSMN-CTC (80 mel, context 2/2, frame skip 3) and DS-TCN-CTC (40 mel,
no context, frame skip 1) -- both with output_dim 2599 (examples/hi_xiaowen/s0/conf/{fsmn,ds_tcn}_ctc.yaml).

Each call is timed with the host clock around the call and a device synchronise, the result's device-to-host copy
included, after a warm-up.  Reported per model and B: p50 / p99 call time, streams served in real time
(B * 0.3 s / p50 call time) and our kernel launches per call.  The card's name and power limit are read in the same
run.  Prints one JSON line.

    python scripts/bench_spotter.py [--batches 1,64,1024] [--calls 100] [--warmup 10]
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

from wekws_b200 import Fbank, KeywordSpotter, _native, init_model, model_config, synth      # noqa: E402

CHUNK = 4800                   # 0.3 s at 16 kHz, the reference demo's chunk (stream_kws_ctc.py:559)
KEYWORDS = {"hi_xiaowen": [5, 9, 17, 23], "nihao_wenwen": [31, 7, 23, 23]}


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def spotter(name: str, B: int, dev: str) -> KeywordSpotter:
    if name == "fsmn_ctc":
        cfg, fb, ctx, skip = model_config("fsmn", input_dim=400, output_dim=2599), Fbank(80), (2, 2), 3
    else:
        cfg, fb, ctx, skip = model_config("ds_tcn", input_dim=40, output_dim=2599, activation="identity"), Fbank(40), None, 1
    torch.manual_seed(777)
    model = synth.randomize_(init_model(cfg)).eval().to(dev)
    return KeywordSpotter(model, KEYWORDS, B, frontend=fb, context=ctx, frame_skip=skip)


def measure(name: str, B: int, calls: int, warmup: int, dev: str) -> dict:
    spot = spotter(name, B, dev)
    audio = synth.pcm_int16(B, CHUNK * 8, seed=B).to(dev)
    chunks = [audio[:, i * CHUNK:(i + 1) * CHUNK] for i in range(8)]
    for i in range(warmup):
        spot(chunks[i % 8]).to_python()
    torch.cuda.synchronize()
    times, launches, activations = [], [], 0
    for i in range(calls):
        n0 = _native.launch_count()
        t0 = time.perf_counter()
        res = spot(chunks[i % 8])
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        launches.append(_native.launch_count() - n0)
        activations += int((res.state == 1).sum())
    t = np.array(times)
    p50, p99 = float(np.percentile(t, 50)), float(np.percentile(t, 99))
    return {"model": name, "streams": B, "calls": calls, "p50_ms": p50 * 1e3, "p99_ms": p99 * 1e3,
            "realtime_streams": B * CHUNK / 16000 / p50, "launches_per_call": sorted(set(launches)),
            "activations": activations}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,64,1024")
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_spotter.py needs a CUDA device")
    if args.calls < 50:
        raise SystemExit("--calls must be >= 50 for a p99")
    dev = "cuda:0"
    rows = [measure(name, int(B), args.calls, args.warmup, dev) for name in ("fsmn_ctc", "ds_tcn_ctc")
            for B in args.batches.split(",")]
    print(json.dumps({"bench": "stream_spotter", "chunk_s": CHUNK / 16000, "card": card(), "results": rows}))


if __name__ == "__main__":
    main()
