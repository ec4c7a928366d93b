"""Raw PCM -> posteriors in one native call (the composition the reference's callers perform by hand:
``feats = accept_wave(wave); logits, cache = model(feats, cache)``, wekws/bin/stream_kws_ctc.py:482-487, and
score.py's dataset front-end + ``model(feats)``, score.py:117-127).

``Pipeline(frontend, model)(pcm, cache)`` goes through ``wekws_pipeline_forward`` of the C ABI: the front-end kernel
and the fused model kernel are launched back to back on the caller's stream with the feature tensor pinned in L2 by
a persisting access-policy window, so the (B, frames, idim) features are produced and consumed on chip.
"""
from __future__ import annotations

from typing import Tuple

import torch

from . import _native
from .frontend import Fbank
from .kws_model import KWSModel, _EMPTY


class Pipeline:
    def __init__(self, frontend: Fbank, model: KWSModel):
        if frontend.feature_dim != model.idim:
            raise ValueError(f"the front-end produces {frontend.feature_dim} features, the model expects {model.idim}")
        self.frontend, self.model = frontend, model
        self._scratch = None

    def __call__(self, pcm: torch.Tensor, in_cache: torch.Tensor = _EMPTY, softmax: bool = False
                 ) -> Tuple[torch.Tensor, torch.Tensor]:
        """pcm (B, N) int16 / float32 CUDA rows at int16 scale -> (posteriors, cache) as ``model(frontend(pcm),
        in_cache)`` returns them: (B, frames, odim) per frame, or with a global / last classifier head one (B, odim) row
        per clip, pooled over its frames.  softmax: over odim, as ``forward_softmax``."""
        m, fe = self.model, self.frontend
        pcm, code, _ = _native.pcm_rows(pcm, "Pipeline", one_d=False, dtype_error=ValueError)
        if m.training:
            raise RuntimeError("wekws_b200.KWSModel is inference-only: call model.eval() first")
        dev = pcm.device
        B, N = pcm.shape
        T = fe.num_frames(N)
        cache, out, out_cache = m._io_tensors(in_cache, B, T, dev)
        if B == 0 or T == 0:
            return out, out_cache
        need = B * T * m.idim
        if self._scratch is None or self._scratch.numel() < need or self._scratch.device != dev:
            self._scratch = torch.empty(need, device=dev, dtype=torch.float32)
        _native.call("wekws_pipeline_forward", fe._handle(dev), m._prepare(dev), pcm, code, B, N, pcm.stride(0),
                     self._scratch, cache, out, out_cache, _native.FWD_SOFTMAX if softmax else 0, device=dev)
        return out, out_cache
