"""wekws_b200 -- H100-native (sm_90a) streaming keyword-spotting forward path for WeKws.

Public surface mirrors the reference (wenet-e2e/wekws):
    init_model, KWSModel     <- wekws/model/kws_model.py
    Fbank, fbank             <- torchaudio.compliance.kaldi.fbank as the reference calls it
    Mfcc, mfcc               <- torchaudio.compliance.kaldi.mfcc  (processor.py:157-166, the mdtc configs' front-end)
    Resample, resample       <- torchaudio.transforms.Resample (processor.py resample(), compute_cmvn_stats.py:50-53)
    CmvnStats, scp_segment   <- tools/compute_cmvn_stats.py: global CMVN statistics and its global_cmvn JSON
    load_cmvn, load_kaldi_cmvn <- wekws/utils/cmvn.py
    Pipeline(frontend, model) <- raw PCM -> posteriors in one native call (stream_kws_ctc.py:482-487 composition)
    patch_reference()        -> makes `wekws.model.kws_model` resolve to this implementation
    det_stats, det_curve     <- wekws/bin/compute_det.py threshold sweep (on the device, bit-exact)
    ctc_prefix_beam_search, ctc_keyword_hits, write_ctc_scores <- wekws/model/loss.py:206-312 + score_ctc.py:198-226
    KeywordSpotter           <- wekws/bin/stream_kws_ctc.py KeyWordSpotter: online CTC keyword spotting, B streams per call
    stream_score_ctc, write_stream_ctc_scores <- wekws/bin/stream_score_ctc.py: streaming decode of a CTC test set
    ctc_det_stats, write_ctc_det_stats <- wekws/bin/compute_det_ctc.py: DET statistics of a CTC score file
    criterion                <- wekws/model/loss.py criterion(): held-out loss / accuracy (max_pooling, ce, ctc)
    context_expansion        <- wekws/dataset/processor.py context_expansion + frame_skip (FSMN / CTC recipes)
    export_native()          -> weight file for the C++ runtime shim (the role of wekws/bin/export_onnx.py)
    export_onnx()            <- wekws/bin/export_onnx.py: the ONNX file (input, cache -> output, r_cache) for the ORT runtime
"""
from .cmvn import load_cmvn, load_kaldi_cmvn
from .cmvn_stats import CmvnStats, scp_segment
from .configs import MODEL_NAMES, model_config
from .frontend import Fbank, Mfcc, Resample, fbank, mfcc, resample
from .kws_model import GlobalCMVN, KWSModel, init_model
from .ctc import (ctc_keyword_hits, ctc_prefix_beam_search, ctc_state, stream_score_ctc, write_ctc_scores,
                  write_stream_ctc_scores)
from .criterion import criterion
from .export import export_native
from .export_onnx import export_onnx
from .overlay import patch_reference
from .pipeline import Pipeline
from .postproc import (context_expansion, ctc_det_stats, det_curve, det_stats, det_thresholds, space_mixed_label,
                       write_ctc_det_stats)
from .spotter import KeywordSpotter, SpotResult

__all__ = ["init_model", "KWSModel", "GlobalCMVN", "Fbank", "fbank", "Mfcc", "mfcc", "load_cmvn", "load_kaldi_cmvn",
           "model_config", "MODEL_NAMES", "patch_reference", "export_native", "export_onnx", "det_stats", "det_curve", "det_thresholds", "context_expansion",
           "Pipeline", "ctc_prefix_beam_search", "ctc_keyword_hits", "ctc_state", "write_ctc_scores",
           "KeywordSpotter", "SpotResult", "stream_score_ctc", "write_stream_ctc_scores", "ctc_det_stats",
           "write_ctc_det_stats", "space_mixed_label", "criterion", "Resample", "resample", "CmvnStats", "scp_segment"]
__version__ = "0.1.0"
