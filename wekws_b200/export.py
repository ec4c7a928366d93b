"""Native weight file for the C++ runtime shim (wekws_b200/runtime/keyword_spotting_b200.h).

The reference ships models to its C++ runtime as ONNX (wekws/bin/export_onnx.py:42-94: inputs ``input``,
``cache`` -> outputs ``output``, ``r_cache``, metadata ``cache_dim`` / ``cache_len``).  The native runtime needs no
graph -- the network is the fused kernels -- only the configuration and the tensors of the reference
``state_dict`` under their reference keys, which is what a ``.wkb`` file holds:

    "WKB1" | int32 version (2) | int32 nconfig | wekws_model_config (nconfig x int32) | int32 ntensors |
    ntensors x ( int32 name_len | name | int64 numel | numel x float32 )        (little endian)
"""
from __future__ import annotations

import struct

import torch

MAGIC, VERSION = b"WKB1", 2


def export_native(model, path: str) -> dict:
    """Writes ``model`` (a wekws_b200.KWSModel, e.g. after load_state_dict of a reference checkpoint) to ``path``.
    Returns the metadata the ONNX exporter would have attached (export_onnx.py:72-77)."""
    if getattr(model, "head", None) is not None:
        raise NotImplementedError(f"export_native: the '{model.head}' classifier head cannot be exported: the runtime "
                                  "shim is frame-level and the .wkb configuration does not carry the head")
    cfg = model._native_config()
    fields = [getattr(cfg, name) for name, _ in cfg._fields_]
    tensors = [(k, v.detach().to(device="cpu", dtype=torch.float32).contiguous())
               for k, v in model.state_dict().items() if not k.endswith("num_batches_tracked")]
    with open(path, "wb") as f:
        f.write(MAGIC)
        f.write(struct.pack("<i", VERSION))
        f.write(struct.pack("<i", len(fields)))
        f.write(struct.pack("<%di" % len(fields), *fields))
        f.write(struct.pack("<i", len(tensors)))
        for name, t in tensors:
            raw = name.encode()
            f.write(struct.pack("<i", len(raw)))
            f.write(raw)
            f.write(struct.pack("<q", t.numel()))
            f.write(t.numpy().tobytes())
    fsmn = getattr(model.backbone, "kind", None) == "fsmn"
    return {"cache_dim": model.backbone.proj_dim if fsmn else model.hdim,
            "cache_len": model.backbone.cache_len if fsmn else getattr(model.backbone, "padding", 0),
            "tensors": len(tensors)}


def read_native(path: str):
    """Parses a .wkb file back into (config fields, {name: tensor}) -- used by the tests."""
    with open(path, "rb") as f:
        data = f.read()
    assert data[:4] == MAGIC, "not a .wkb file"
    off = 4
    (version,) = struct.unpack_from("<i", data, off); off += 4
    assert version == VERSION
    (nconfig,) = struct.unpack_from("<i", data, off); off += 4
    fields = struct.unpack_from("<%di" % nconfig, data, off); off += 4 * nconfig
    (n,) = struct.unpack_from("<i", data, off); off += 4
    out = {}
    for _ in range(n):
        (ln,) = struct.unpack_from("<i", data, off); off += 4
        name = data[off:off + ln].decode(); off += ln
        (numel,) = struct.unpack_from("<q", data, off); off += 8
        out[name] = torch.frombuffer(bytearray(data[off:off + 4 * numel]), dtype=torch.float32).clone(); off += 4 * numel
    assert off == len(data)
    return fields, out
