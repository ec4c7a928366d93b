"""Cost of scoring a CTC test set with the streaming decoder (wekws_b200.stream_score_ctc, ctc_stream_score_kernel):
a synthetic test set of peaky V = 2599 posteriors (the output_dim of examples/hi_xiaowen/s0/conf/*_ctc.yaml), in
batches of 256 utterances of up to 1000 frames, two keywords.

Each call is timed with the host clock around the call and a device synchronise after a warm-up; the call includes its
one read of the activation counts.  Reported: p50 / p99 time per batch, utterance-hours decoded per second
(frames * frame_skip * 10 ms / p50) and the HBM rate of the probability read (valid rows * V * 4 bytes / p50; every
valid row is read once).  Beside it, the oracle restatement of the reference's Python loop
(oracle/kws_stream_score_oracle.py) on one host core for a few utterances, extrapolated to the batch.  The card's name
and power limit are read in the same run.  Prints one JSON line.

    python scripts/bench_stream_score.py [--batch 256] [--max-frames 1000] [--repeats 30] [--oracle-utts 4]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.kws_stream_score_oracle import stream_score      # noqa: E402
from scripts.bench_spotter import card                       # noqa: E402
from wekws_b200 import _native, stream_score_ctc             # noqa: E402

V = 2599
KEYWORDS = {"hi_xiaowen": [5, 9, 17, 23], "nihao_wenwen": [31, 7, 23, 23]}


def test_set(B, max_frames, seed, dev):
    """Peaky posteriors: mostly blank, keyword spellings (2 frames per token) at random places, a few frames owned by
    a token outside the keywords; lengths uniform in max_frames / 5 .. max_frames."""
    rng = np.random.RandomState(seed)
    lens = rng.randint(max_frames // 5, max_frames + 1, size=B).astype(np.int32)
    dom = np.zeros((B, max_frames), dtype=np.int64)
    seqs = list(KEYWORDS.values())
    for b in range(B):
        t = int(rng.randint(0, 40))
        while t < lens[b]:
            for tok in seqs[int(rng.randint(len(seqs)))]:
                dom[b, t:t + 2] = tok
                t += 3
            t += int(rng.randint(20, 120))
    dom[rng.rand(B, max_frames) < 0.03] = 1500
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(B, max_frames, V, generator=g, device=dev) * 0.5
    x.scatter_add_(2, torch.from_numpy(dom).to(dev).unsqueeze(-1), torch.full((B, max_frames, 1), 9.0, device=dev))
    return x.softmax(-1), torch.from_numpy(lens)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--max-frames", type=int, default=1000)
    ap.add_argument("--frame-skip", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-utts", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream_score.py needs a CUDA device")
    dev = "cuda:0"
    probs, lens = test_set(args.batch, args.max_frames, 7, dev)
    for _ in range(args.warmup):
        stream_score_ctc(probs, lens, KEYWORDS, frame_skip=args.frame_skip)
    torch.cuda.synchronize()
    times, launches = [], set()
    for _ in range(args.repeats):
        n0 = _native.launch_count()
        t0 = time.perf_counter()
        res = stream_score_ctc(probs, lens, KEYWORDS, frame_skip=args.frame_skip)
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        launches.add(_native.launch_count() - n0)
    t = np.array(times)
    p50, p99 = float(np.percentile(t, 50)), float(np.percentile(t, 99))
    frames = int(lens.sum())
    audio_h = frames * args.frame_skip * 0.01 / 3600
    nbytes = frames * V * 4
    # the reference's loop, restated, on one host core for a few utterances
    torch.set_num_threads(1)
    n = min(args.oracle_utts, args.batch)
    host = probs[:n].cpu()
    t0 = time.perf_counter()
    for b in range(n):
        stream_score(host[b, :int(lens[b])], KEYWORDS, frame_skip=args.frame_skip)
    host_s = time.perf_counter() - t0
    host_frames = int(lens[:n].sum())
    host_batch_s = host_s / host_frames * frames
    print(json.dumps({
        "bench": "stream_score_ctc", "card": card(), "V": V, "batch": args.batch, "max_frames": args.max_frames,
        "frames": frames, "frame_skip": args.frame_skip, "repeats": args.repeats, "p50_ms": p50 * 1e3,
        "p99_ms": p99 * 1e3, "utterance_hours_per_s": audio_h / p50, "prob_read_gb": nbytes / 1e9,
        "prob_read_gb_per_s": nbytes / p50 / 1e9, "launches_per_call": sorted(launches),
        "activations": int(res.count.sum()),
        "host_oracle": {"utterances": n, "frames": host_frames, "seconds": host_s,
                        "extrapolated_batch_s": host_batch_s, "extrapolated_speedup": host_batch_s / p50}}))


if __name__ == "__main__":
    main()
