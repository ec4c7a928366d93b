"""ctypes binding of the C-ABI shared library (include/wekws_b200.h), and the one place that knows how a native call
is made: ``call`` for the stream-taking entry points, ``invoke`` / ``create`` for the others, ``pcm_rows`` /
``host_lengths`` for the PCM input every audio entry point accepts, ``DeviceHandles`` for per-device native objects.

The library is built in-tree (``python -c 'import __graft_entry__ as g; g.build()'`` or
``make -C wekws_b200/csrc``).  There is NO fallback: if the library is missing or a call
fails, a RuntimeError carrying ``wekws_last_error()`` is raised.
"""
from __future__ import annotations

import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# WEKWS_B200_LIB: development override (A/B of two builds of the same ABI); the product default is the in-tree library
LIB_PATH = os.environ.get("WEKWS_B200_LIB") or os.path.join(_HERE, "libwekws_b200.so")

# enums (include/wekws_b200.h)
BACKBONE_MDTC, BACKBONE_TCN, BACKBONE_DSTCN, BACKBONE_GRU, BACKBONE_FSMN = 0, 1, 2, 3, 4
ACT_IDENTITY, ACT_SIGMOID = 0, 1
PCM_S16, PCM_F32 = 0, 1
HEAD_LINEAR, HEAD_GLOBAL, HEAD_LAST = 0, 1, 2
FWD_SOFTMAX = 1
ABI_VERSION = 19

# limits (include/wekws_b200.h #defines)
CTC_MAX_PREFIX, CTC_MAX_PATH_BEAM, CTC_MAX_SCORE_BEAM = 64, 20, 3
CRITERION_MAX_LABEL = 511        # one thread per extended-label state (2 L + 1 <= 1023)

# records the kernels write (numpy dtypes of wekws_ctc_spot_result / wekws_ctc_stream_detection)
SPOT_RESULT_DTYPE = [("score", "<f8"), ("state", "<i4"), ("keyword", "<i4"), ("start", "<i4"), ("end", "<i4"),
                     ("overflow", "<i4"), ("reserved", "<i4")]
SPOT_RESULT_BYTES = 32
STREAM_DETECTION_DTYPE = [("score", "<f8"), ("keyword", "<i4"), ("start", "<i4"), ("end", "<i4"), ("frame", "<i4")]
STREAM_DETECTION_BYTES = 24
THRESHOLD_EVENT_DTYPE = [("frame", "<i8"), ("keyword", "<i4"), ("score", "<f4")]      # wekws_threshold_event
THRESHOLD_EVENT_BYTES = 16


class FbankConfig(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("frame_length", C.c_int32), ("frame_shift", C.c_int32),
                ("n_fft", C.c_int32), ("num_mel_bins", C.c_int32), ("preemphasis", C.c_float),
                ("remove_dc", C.c_int32), ("log_floor", C.c_float)]


class ModelConfig(C.Structure):
    _fields_ = [("backbone", C.c_int32), ("idim", C.c_int32), ("hdim", C.c_int32), ("odim", C.c_int32),
                ("num_layers", C.c_int32), ("num_stack", C.c_int32), ("stack_size", C.c_int32),
                ("kernel_size", C.c_int32), ("activation", C.c_int32), ("norm_var", C.c_int32),
                ("fsmn_input_affine_dim", C.c_int32), ("fsmn_linear_dim", C.c_int32), ("fsmn_proj_dim", C.c_int32),
                ("fsmn_left_order", C.c_int32), ("fsmn_right_order", C.c_int32),
                ("fsmn_output_affine_dim", C.c_int32)]


# name -> (restype, argtypes); every symbol include/wekws_b200.h declares
SIGNATURES = {
    "wekws_last_error": (C.c_char_p, []),
    "wekws_abi_version": (C.c_int, []),
    "wekws_launch_count": (C.c_uint64, []),
    "wekws_fbank_create": (C.c_int, [C.POINTER(FbankConfig), C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]),
    "wekws_fbank_destroy": (None, [C.c_void_p]),
    "wekws_fbank_num_frames": (C.c_int64, [C.c_void_p, C.c_int64]),
    "wekws_fbank_num_mel_bins": (C.c_int, [C.c_void_p]),
    "wekws_fbank_feature_dim": (C.c_int, [C.c_void_p]),
    "wekws_fbank_set_mfcc": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wekws_fbank_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "wekws_fbank_forward_dither": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float,
                                             C.c_uint64, C.c_void_p]),
    "wekws_dither_noise": (C.c_int, [C.c_uint64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p]),
    "wekws_spec_aug": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                 C.c_void_p]),
    "wekws_reverb": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p,
                               C.c_int64, C.c_void_p]),
    "wekws_add_noise": (C.c_int, [C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]),
    "wekws_model_create": (C.c_int, [C.POINTER(ModelConfig), C.POINTER(C.c_void_p)]),
    "wekws_model_destroy": (None, [C.c_void_p]),
    "wekws_model_padding": (C.c_int, [C.c_void_p]),
    "wekws_model_set_tensor": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "wekws_model_set_head": (C.c_int, [C.c_void_p, C.c_int]),
    "wekws_model_pack": (C.c_int, [C.c_void_p]),
    "wekws_model_finalize": (C.c_int, [C.c_void_p]),
    "wekws_model_set_precision": (C.c_int, [C.c_void_p, C.c_int]),
    "wekws_model_uses_tensor_cores": (C.c_int, [C.c_void_p, C.c_int64]),
    "wekws_model_uses_tensor_cores_bt": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64]),
    "wekws_model_packed_floats": (C.c_int64, [C.c_void_p, C.c_int]),
    "wekws_model_packed_copy": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int64]),
    "wekws_model_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int64, C.c_int64, C.c_uint32, C.c_void_p]),
    "wekws_det_stats": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_threshold_spot_state_bytes": (C.c_int64, []),
    "wekws_threshold_spot": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int,
                                       C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_ctc_state_bytes": (C.c_int64, []),
    "wekws_ctc_prefix_beam_search": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int,
                                               C.c_int, C.c_int, C.c_int64, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p]),
    "wekws_ctc_keyword_hit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "wekws_ctc_spot_state_bytes": (C.c_int64, []),
    "wekws_ctc_spot": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_int,
                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_ctc_stream_score": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, C.c_int,
                                         C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_stream_pcm": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]),
    "wekws_stream_context": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_void_p]),
    "wekws_context_expand_frames": (C.c_int64, [C.c_int64, C.c_int, C.c_int]),
    "wekws_context_expand": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p, C.c_int64, C.c_void_p]),
    "wekws_criterion_max_pooling_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "wekws_criterion_max_pooling": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_int,
                                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_criterion_ce_workspace_bytes": (C.c_int64, [C.c_int64]),
    "wekws_criterion_ce": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_criterion_ctc_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int64, C.c_int]),
    "wekws_criterion_ctc": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_int64,
                                      C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_criterion_max_pooling_train": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                                    C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_void_p]),
    "wekws_criterion_max_pooling_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int,
                                                       C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_criterion_ce_train": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_criterion_ce_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "wekws_criterion_ctc_train": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                            C.c_int64, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p]),
    "wekws_criterion_ctc_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p,
                                               C.c_int64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_train_num_params": (C.c_int, [C.c_void_p]),
    "wekws_train_saved_floats": (C.c_int64, [C.c_void_p, C.c_int64, C.c_int64]),
    "wekws_train_backward_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int64, C.c_int64]),
    "wekws_train_backward_launches": (C.c_int, [C.c_void_p]),
    "wekws_train_workspace_bytes": (C.c_int64, [C.c_void_p, C.c_int64, C.c_int64, C.c_int]),
    "wekws_train_forward_launches": (C.c_int, [C.c_void_p]),
    "wekws_train_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "wekws_train_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int, C.c_int64, C.c_int64,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_model_load_params": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]),
    "wekws_model_train_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                            C.c_int64, C.c_void_p]),
    "wekws_model_backward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                       C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "wekws_dropout_mask": (C.c_int, [C.c_uint64, C.c_int64, C.c_int64, C.c_int64, C.c_int, C.c_uint32, C.c_void_p,
                                     C.c_void_p]),
    "wekws_pipeline_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64,
                                         C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_uint32, C.c_void_p]),
    "wekws_resample_create": (C.c_int, [C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "wekws_resample_destroy": (None, [C.c_void_p]),
    "wekws_resample_output_length": (C.c_int64, [C.c_void_p, C.c_int64]),
    "wekws_resample_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int64, C.c_int64, C.c_int64, C.c_void_p,
                                         C.c_void_p, C.c_int64, C.c_int64, C.c_void_p]),
    "wekws_grad_clip_workspace_bytes": (C.c_int64, [C.c_int, C.c_int64]),
    "wekws_grad_clip_launches": (C.c_int, [C.c_int]),
    "wekws_grad_clip": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]),
    "wekws_adam_step_launches": (C.c_int, [C.c_int]),
    "wekws_adam_step": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_void_p]),
    "wekws_cmvn_stats_workspace_bytes": (C.c_int64, [C.c_int64, C.c_int]),
    "wekws_cmvn_stats_accumulate": (C.c_int, [C.c_void_p, C.c_int64, C.c_int64, C.c_int, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p]),
}

_lib = None


def lib() -> C.CDLL:
    """Loads libwekws_b200.so once; raises if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"wekws_b200: native library {LIB_PATH} is not built. Run "
                "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). "
                "There is no CPU or PyTorch fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)      # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        got = l.wekws_abi_version()
        if got != ABI_VERSION:
            raise RuntimeError(f"wekws_b200: ABI version mismatch (library {got}, binding {ABI_VERSION})")
        _lib = l
    return _lib


def last_error() -> str:
    return lib().wekws_last_error().decode("utf-8", "replace")


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"wekws_b200: {what} failed (status {rc}): {last_error()}")


def launch_count() -> int:
    return int(lib().wekws_launch_count())


def call(name: str, *args, device: torch.device) -> None:
    """Runs the stream-taking entry point ``name(*args, stream)`` on ``device``'s current stream with ``device``
    current (no switch when it already is).  A tensor argument is passed as its data pointer; None (NULL), integers
    and ctypes objects as they are.  Raises RuntimeError with the library's message on a non-zero status."""
    fn = getattr(_lib if _lib is not None else lib(), name)
    args = [a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]
    stream = torch.cuda.current_stream(device).cuda_stream
    if torch.cuda.current_device() == device.index:
        rc = fn(*args, stream)
    else:
        with torch.cuda.device(device):
            rc = fn(*args, stream)
    if rc != 0:
        check(rc, name)


def invoke(name: str, *args, what: str = None) -> None:
    """Runs a status-returning entry point that takes no stream (set-up calls), arguments as ``call`` takes them;
    ``what`` names it in the error (default: ``name``)."""
    check(getattr(lib(), name)(*[a.data_ptr() if isinstance(a, torch.Tensor) else a for a in args]), what or name)


def create(name: str, *args) -> C.c_void_p:
    """A new native object from ``name(*args, &handle)`` (the ``*_create`` entry points)."""
    h = C.c_void_p()
    invoke(name, *args, C.byref(h))
    return h


_PCM_CODES = {torch.int16: PCM_S16, torch.float32: PCM_F32}


def pcm_rows(pcm: torch.Tensor, what: str, one_d: bool = True, dtype_error=TypeError):
    """Checks PCM input: int16 or float32 samples at int16 scale on a CUDA device, (B, N) rows or, with ``one_d``, one
    (N,) row.  Returns (the (B, N) rows with unit inner stride, their PCM_* code, whether an (N,) input was lifted to
    one row).  ``what`` names the entry point in the error for a CPU tensor; another dtype raises ``dtype_error``."""
    if not pcm.is_cuda:
        raise RuntimeError(f"wekws_b200.{what} runs on CUDA (sm_90a) only; got a CPU tensor (no CPU fallback)")
    lifted = one_d and pcm.dim() == 1
    if lifted:
        pcm = pcm.unsqueeze(0)
    if pcm.dim() != 2:
        raise ValueError("pcm must be (N,) or (B, N)" if one_d else "pcm must be (B, N)")
    code = _PCM_CODES.get(pcm.dtype)
    if code is None:
        raise dtype_error(f"pcm must be int16 or float32, got {pcm.dtype}")
    if pcm.stride(1) != 1:
        pcm = pcm.contiguous()
    return pcm, code, lifted


def host_lengths(lengths, B: int, N: int) -> list:
    """Valid samples per row given on the host (a sequence or tensor of B ints in 0..N) as a list of ints."""
    lens = [int(n) for n in (lengths.tolist() if isinstance(lengths, torch.Tensor) else lengths)]
    if len(lens) != B or any(n < 0 or n > N for n in lens):
        raise ValueError(f"lengths must be {B} values in 0..{N}")
    return lens


class DeviceHandles:
    """Base of the objects that keep one native object per CUDA device: ``_handle(dev)`` makes it on first use with
    ``_create()`` and then ``_configure(handle)``, both on that device; the ``_DESTROY`` entry point frees them all
    when the owner goes."""
    _DESTROY = ""

    def _create(self) -> C.c_void_p:
        raise NotImplementedError

    def _configure(self, handle) -> None:
        """Hook for subclasses: extra native configuration of a freshly created handle."""

    def _handle(self, dev: torch.device) -> C.c_void_p:
        handles = self.__dict__.setdefault("_handles", {})
        h = handles.get(dev)
        if h is None:
            with torch.cuda.device(dev):
                h = self._create()
                self._configure(h)
            handles[dev] = h
        return h

    def __del__(self):
        for h in self.__dict__.get("_handles", {}).values():
            try:
                getattr(lib(), self._DESTROY)(h)
            except Exception:
                pass
