"""Shared description of the utterance-level classifier-head cases (oracle/make_head_golden.py and
tests/test_classifier_heads.py).  Kept apart from cases.MODEL_CASES: those tests assume per-frame output."""
import contextlib
import io

from wekws_b200 import synth
from wekws_b200.configs import model_config

# case -> (config name, classifier type, output_dim, input_dim)
HEAD_CASES = {
    # examples/speechcommand_v1/s0/conf/mdtc.yaml: the flagship MDTC, 80-ceps MFCC, 11 outputs, classifier global
    "mdtc_global": ("mdtc", "global", 11, 80),
    "mdtc_last": ("mdtc", "last", 11, 80),
    "mdtc_small_last": ("mdtc_small", "last", 5, 40),      # hidden 32: the FP32 conv kernel
    "tcn_global": ("tcn", "global", 3, 80),
}
HEAD_CHUNKS = (40, 17, 1)      # streamed back to back, cache carried
HEAD_B = 2                     # streams of the chunked and whole-utterance calls
FULL_T = 300                   # one whole-utterance call: three internal time-chunks of the tensor-core kernel
BATCH_B, BATCH_T = 8, 98       # a batch of 1 s clips
FULL_SEED, BATCH_SEED = 510, 520   # synth.features seeds of the two long inputs


def head_config(case: str) -> dict:
    name, head, odim, idim = HEAD_CASES[case]
    cfg = model_config(name, input_dim=idim, output_dim=odim)
    cfg["classifier"] = dict(type=head, dropout=0.5)
    return cfg


def build_head_model(case: str, factory, seed: int = 777):
    """Instantiates `factory` (reference or wekws_b200 init_model) with the project's synthetic weights."""
    import torch
    cfg = head_config(case)
    with contextlib.redirect_stdout(io.StringIO()):
        torch.manual_seed(seed)
        model = factory(cfg)
    synth.randomize_(model, seed=seed)
    model.eval()
    return cfg, model
