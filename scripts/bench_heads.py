"""Throughput of the speech-command recipe (examples/speechcommand_v1/s0/conf/mdtc.yaml): B one-second int16 clips
-> Mfcc(80, 80) -> MDTC (hidden 64, 4 x 4, k = 5) with the `global` head, 11 outputs.

For comparison the same preprocessing and backbone weights with the per-frame linear head run on the same features in
the same process, the arms alternating: with 11 outputs (output (B, T, 11); the FP32 conv kernel, since the
tensor-core kernel's per-frame classifier takes at most 8) and with 8 outputs (the same tensor-core kernel as the
head).  Times are CUDA events around `reps` back-to-back calls after a warm-up; the card's name and power limit are
read in the same run.  Prints one JSON line.

    python scripts/bench_heads.py [--batch 1024] [--reps 50] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from wekws_b200 import Mfcc, init_model, model_config, synth      # noqa: E402


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def timed(fn, reps: int) -> float:
    """Seconds per call: CUDA events around `reps` calls."""
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / 1e3 / reps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_heads.py needs a CUDA device")
    dev = "cuda:0"
    cfg = model_config("mdtc", output_dim=11)
    cfg["classifier"] = dict(type="global", dropout=0.5)
    torch.manual_seed(777)
    head = synth.randomize_(init_model(cfg)).eval().to(dev)

    def linear_twin(odim):
        lin = init_model(model_config("mdtc", output_dim=odim)).eval()
        with torch.no_grad():
            sd = head.state_dict()
            for k, v in lin.state_dict().items():
                if not k.startswith("classifier."):
                    v.copy_(sd[k].cpu())
        synth.randomize_(lin.classifier, seed=778)
        return lin.to(dev)
    # 11 outputs exceed the per-frame classifier of the tensor-core kernel (odim <= 8): that model runs the FP32 conv
    # kernel.  The 8-output twin runs the same tensor-core backbone as the head model.
    lin, lin8 = linear_twin(11), linear_twin(8)

    pcm = synth.pcm_int16(args.batch, 16000, seed=1).to(dev)
    fe = Mfcc(80, 80)
    feats = fe(pcm)
    T = feats.size(1)
    arms = {
        "global_head": lambda: head(feats),
        "linear_head": lambda: lin(feats),
        "linear_head_8_outputs": lambda: lin8(feats),
        "global_head_pcm": lambda: head(fe(pcm)),      # front-end included
    }
    for fn in arms.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, args.reps))
    best = {k: min(v) for k, v in times.items()}
    audio_s = args.batch * 16000 / 16000.0
    res = {"workload": "speechcommand_mdtc_global", "batch": args.batch, "frames": T, "card": card(),
           "method": f"CUDA events, {args.rounds} alternating rounds x {args.reps} calls, best round",
           "utt_per_s": {k: args.batch / t for k, t in best.items()},
           "audio_hours_per_s": {k: audio_s / 3600.0 / t for k, t in best.items()},
           "ms_per_call": {k: 1e3 * t for k, t in best.items()},
           "ms_per_call_all_rounds": {k: [round(1e3 * t, 4) for t in v] for k, v in times.items()},
           "tensor_cores": {"global_head": head.uses_tensor_cores(T), "linear_head": lin.uses_tensor_cores(T),
                            "linear_head_8_outputs": lin8.uses_tensor_cores(T)},
           "head_over_linear_time": best["global_head"] / best["linear_head"],
           "head_over_linear_8_outputs_time": best["global_head"] / best["linear_head_8_outputs"]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
