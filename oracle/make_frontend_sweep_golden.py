"""Generates tests/golden/frontend_sweep.npz from torchaudio for every row of tests/test_frontend_sweep.py:

    python oracle/make_frontend_sweep_golden.py

For each row it runs torchaudio.compliance.kaldi.fbank / .mfcc, with that row's options, dither 0 and energy_floor 0,
on the pins' waveform (tests/test_frontend_sweep.py pin_wave) and stores the float32 output under the row's id, with
the waveform's absolute sum (the test regenerates the waveform and checks it against that).  The test then pins the
oracle's front-end options to these outputs where torchaudio is not installed.
TEST INFRASTRUCTURE ONLY.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.test_frontend_sweep import ROW_IDS, _kaldi_call, pin_wave          # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "frontend_sweep.npz")


def main() -> None:
    wav = pin_wave()
    arrays = {"wave_abs_sum": np.float64(wav.double().abs().sum())}
    for row in ROW_IDS:
        arrays[row] = _kaldi_call(row, wav).numpy()
        print(row, arrays[row].shape)
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
