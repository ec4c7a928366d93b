"""ONNX-contract exporter: the file the reference's C++ runtime loads (runtime/core/kws/keyword_spotting.cc:28-95).

The reference produces it with ``torch.onnx.export`` + the ``onnx`` package (wekws/bin/export_onnx.py:42-94); neither
the tracer nor ``onnx`` is needed here: the network of a reference checkpoint is known in closed form (the same folded
eval-mode math the fused kernels run, SURVEY.md section 8 "folded per-block math"), so this module writes the
``ModelProto`` directly in protobuf wire format.  The contract that keyword_spotting.cc relies on is kept exactly:

* inputs  ``input``  (1, T, idim) float32, T dynamic            (export_onnx.py:61, 64)
          ``cache``  (1, hdim, padding) float32 -- FSMN: (1, proj_dim, cache_len, num_layers)   (:55-60)
* outputs ``output`` (1, T, odim), ``r_cache`` (same shape as ``cache``)                         (:65)
* opset 13, metadata_props ``cache_dim`` = hdim, ``cache_len`` = backbone.padding                (:67, :72-77)
* ``softmax=True`` is the CTC export (``model.forward = model.forward_softmax``, :46-48)

BatchNorm is folded into the preceding convolution (what ``do_constant_folding=True`` does to an eval-mode model).
GRU models have no ``backbone.padding`` and cannot be exported by the reference either (:57 raises) -- same here.

The graph is plain opset-13 operators (Sub, Mul, MatMul, Add, Relu, Transpose, Concat, Slice, Conv, Squeeze,
Unsqueeze, Sigmoid, Softmax); tests/onnx_mini.py decodes the file again and evaluates it against the oracle.
"""
from __future__ import annotations

from typing import Dict, Iterable, List, Sequence, Tuple

import numpy as np
import torch

OPSET = 13
IR_VERSION = 7                  # the IR version onnx 1.8 - 1.10 pair with opset 13
FLOAT, INT64 = 1, 7             # TensorProto.DataType


# ----------------------------------------------------------------------------------------------- protobuf wire format
def _varint(v: int) -> bytes:
    if v < 0:
        v += 1 << 64            # int64 two's complement, 10 bytes
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        if v:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _f_varint(field: int, v: int) -> bytes:
    return _varint(field << 3) + _varint(v)


def _f_bytes(field: int, payload: bytes) -> bytes:
    return _varint((field << 3) | 2) + _varint(len(payload)) + payload


def _f_str(field: int, s: str) -> bytes:
    return _f_bytes(field, s.encode())


def _tensor(name: str, arr: np.ndarray) -> bytes:
    """TensorProto: dims = 1, data_type = 2, name = 8, raw_data = 9 (little endian)."""
    if arr.dtype == np.float32:
        dt = FLOAT
    elif arr.dtype == np.int64:
        dt = INT64
    else:
        raise TypeError(arr.dtype)
    b = b"".join(_f_varint(1, int(d)) for d in arr.shape)
    return b + _f_varint(2, dt) + _f_str(8, name) + _f_bytes(9, np.ascontiguousarray(arr).astype(arr.dtype.newbyteorder("<")).tobytes())


def _attr_int(name: str, v: int) -> bytes:          # AttributeProto: name = 1, i = 3, type = 20 (INT = 2)
    return _f_str(1, name) + _f_varint(3, v) + _f_varint(20, 2)


def _attr_ints(name: str, vs: Iterable[int]) -> bytes:   # ints = 8, type INTS = 7
    return _f_str(1, name) + b"".join(_f_varint(8, int(v)) for v in vs) + _f_varint(20, 7)


def _value_info(name: str, shape: Sequence) -> bytes:
    """ValueInfoProto{name = 1, type = 2: TypeProto{tensor_type = 1: {elem_type = 1, shape = 2: {dim = 1*}}}}."""
    dims = b""
    for d in shape:
        dims += _f_bytes(1, _f_str(2, d) if isinstance(d, str) else _f_varint(1, int(d)))
    ttype = _f_varint(1, FLOAT) + _f_bytes(2, dims)
    return _f_str(1, name) + _f_bytes(2, _f_bytes(1, ttype))


class _Graph:
    """Accumulates nodes and initializers; value names are generated."""

    def __init__(self):
        self.nodes: List[bytes] = []
        self.inits: List[bytes] = []
        self._n = 0

    def name(self, hint: str) -> str:
        self._n += 1
        return f"{hint}_{self._n}"

    def const(self, arr, hint: str = "c") -> str:
        if isinstance(arr, torch.Tensor):
            arr = arr.detach().cpu().numpy()
        arr = np.asarray(arr)
        if arr.dtype not in (np.float32, np.int64):
            arr = arr.astype(np.float32)
        n = self.name(hint)
        self.inits.append(_tensor(n, arr))
        return n

    def node(self, op: str, inputs: Sequence[str], attrs: Sequence[bytes] = (), out: str = None, nout: int = 1):
        """NodeProto: input = 1, output = 2, name = 3, op_type = 4, attribute = 5."""
        outs = [out] if out is not None else [self.name(op.lower()) for _ in range(nout)]
        b = b"".join(_f_str(1, i) for i in inputs) + b"".join(_f_str(2, o) for o in outs)
        b += _f_str(3, self.name("n")) + _f_str(4, op) + b"".join(_f_bytes(5, a) for a in attrs)
        self.nodes.append(b)
        return outs[0] if nout == 1 else outs

    def slice(self, x: str, start: int, end: int, axis: int) -> str:
        i64 = lambda v: self.const(np.array([v], dtype=np.int64), "i")
        return self.node("Slice", [x, i64(start), i64(end), i64(axis)])

    def conv(self, x: str, w: torch.Tensor, b: torch.Tensor, dilation: int = 1, groups: int = 1) -> str:
        attrs = [_attr_ints("dilations", [dilation]), _attr_int("group", groups),
                 _attr_ints("kernel_shape", [w.shape[2]]), _attr_ints("pads", [0, 0]), _attr_ints("strides", [1])]
        return self.node("Conv", [x, self.const(w, "w"), self.const(b, "b")], attrs)

    def linear(self, x: str, w: torch.Tensor, b: torch.Tensor = None) -> str:
        """x (.., in) @ w.T (+ b)  -- nn.Linear as MatMul + Add, what the tracer emits for 3-D inputs."""
        y = self.node("MatMul", [x, self.const(w.t().contiguous(), "w")])
        return y if b is None else self.node("Add", [y, self.const(b, "b")])


# --------------------------------------------------------------------------------------------------------- BN folding
def _fold(sd: Dict[str, torch.Tensor], conv: str, bn: str) -> Tuple[torch.Tensor, torch.Tensor]:
    """Conv1d followed by eval-mode BatchNorm1d (eps 1e-5) as one convolution, in float64 then rounded once."""
    w, b = sd[conv + ".weight"].double(), sd[conv + ".bias"].double()
    s = sd[bn + ".weight"].double() / torch.sqrt(sd[bn + ".running_var"].double() + 1e-5)
    t = sd[bn + ".bias"].double() - sd[bn + ".running_mean"].double() * s
    return (w * s.view(-1, 1, 1)).float(), (b * s + t).float()


def _cat_cache(g: _Graph, cache: str, x: str, off: int, pad: int) -> Tuple[str, str]:
    """y = cat(cache[:, :, off:off+pad], x); new slice = y[:, :, -pad:]   (mdtc.py:108-113 == tcn.py:49-54)."""
    y = g.node("Concat", [g.slice(cache, off, off + pad, 2), x], [_attr_int("axis", 2)])
    return y, g.slice(y, -pad, np.iinfo(np.int64).max, 2)


def _mdtc(g: _Graph, sd, bb, x: str, cache: str, C: int) -> Tuple[str, str]:
    k = bb.kernel_size
    blocks = [("backbone.preprocessor", 1)] + [(f"backbone.blocks.{s}.res_blocks.{l}", 2 ** l)
                                               for s in range(bb.num_stack) for l in range(bb.stack_size)]
    off, caches, outs = 0, [], []
    for i, (p, d) in enumerate(blocks):
        pad = d * (k - 1)
        y, c = _cat_cache(g, cache, x, off, pad)
        caches.append(c)
        off += pad
        o = g.conv(y, *_fold(sd, p + ".conv1.conv", p + ".conv1.bn"), dilation=d, groups=C)       # mdtc.py:56-57
        o = g.node("Relu", [g.conv(o, *_fold(sd, p + ".conv1.pointwise", p + ".bn1"))])          # :58, :115
        o = g.conv(o, *_fold(sd, p + ".conv2", p + ".bn2"))                                       # :116
        x = g.node("Relu", [g.node("Add", [o, x])])                                               # :117-120
        if i > 0 and i % bb.stack_size == 0:
            outs.append(x)                                                                        # :266
    y = outs[0]
    for o in outs[1:]:
        y = g.node("Add", [y, o])                                                                 # :270-273
    return y, g.node("Concat", caches, [_attr_int("axis", 2)])


def _tcn(g: _Graph, sd, bb, x: str, cache: str, C: int) -> Tuple[str, str]:
    k, off, caches = bb.kernel_size, 0, []
    for i in range(bb.num_layers):
        d, p = 2 ** i, f"backbone.network.{i}.cnn"
        pad = (k - 1) * d
        y, c = _cat_cache(g, cache, x, off, pad)
        caches.append(c)
        off += pad
        if bb.ds:                                                                                 # tcn.py:101-114
            y = g.node("Relu", [g.conv(y, *_fold(sd, p + ".0", p + ".1"), dilation=d, groups=C)])
            y = g.node("Relu", [g.conv(y, *_fold(sd, p + ".3", p + ".4"))])
        else:                                                                                     # tcn.py:75-84
            y = g.node("Relu", [g.conv(y, *_fold(sd, p + ".0", p + ".1"), dilation=d)])
        x = g.node("Add", [y, x])                                                                 # tcn.py:60
    return x, g.node("Concat", caches, [_attr_int("axis", 2)])


def _fsmn(g: _Graph, sd, bb, x: str, cache: str) -> Tuple[str, str]:
    """fsmn.py:458-495.  The memory block (fsmn.py:223-251) -- identity tap + left FIR + right FIR over
    cat(cache, p) -- is one depthwise convolution with lorder + rorder taps."""
    lo, ro, L, P = bb.lorder, bb.rorder, bb.fsmn_layers, bb.proj_dim
    pad = lo - 1 + ro
    lin = lambda h, p, bias=True: g.linear(h, sd[p + ".weight"], sd[p + ".bias"] if bias else None)
    h = lin(x, "backbone.in_linear1.linear")
    h = g.node("Relu", [lin(h, "backbone.in_linear2.linear")])
    axes3 = g.const(np.array([3], dtype=np.int64), "i")
    new = []
    for l in range(L):
        pre = f"backbone.fsmn.{l}."
        p = g.node("Transpose", [lin(h, pre + "0.linear", bias=False)], [_attr_ints("perm", [0, 2, 1])])
        c = g.node("Squeeze", [g.slice(cache, l, l + 1, 3), axes3])
        cat = g.node("Concat", [c, p], [_attr_int("axis", 2)])
        new.append(g.node("Unsqueeze", [g.slice(cat, -pad, np.iinfo(np.int64).max, 2), axes3]))
        w = torch.zeros(P, 1, lo + ro)
        w[:, 0, :lo] = sd[pre + "1.conv_left.weight"].reshape(P, lo)
        w[:, 0, lo - 1] += 1.0
        w[:, 0, lo:] = sd[pre + "1.conv_right.weight"].reshape(P, ro)
        o = g.conv(cat, w, torch.zeros(P), groups=P)
        o = g.node("Transpose", [o], [_attr_ints("perm", [0, 2, 1])])
        h = g.node("Relu", [lin(o, pre + "2.linear")])
    h = lin(lin(h, "backbone.out_linear1.linear"), "backbone.out_linear2.linear")
    return h, g.node("Concat", new, [_attr_int("axis", 3)])


def export_onnx(model, path: str, softmax: bool = False) -> dict:
    """Writes ``model`` (a wekws_b200.KWSModel holding a reference state_dict) as the ONNX file of
    wekws/bin/export_onnx.py.  Returns the metadata that was attached."""
    bb = model.backbone
    kind = getattr(bb, "kind", None)
    if getattr(model, "head", None) is not None:
        raise NotImplementedError(f"export_onnx: the '{model.head}' classifier head is not exported yet; the graph "
                                  "here is the frame-level (input, cache) -> (output, r_cache) contract")
    if kind not in ("mdtc", "tcn", "ds_tcn", "fsmn"):
        raise NotImplementedError("export_onnx: the ONNX contract needs `backbone.padding` (mdtc / tcn / ds_tcn / fsmn); "
                                  "the reference's exporter fails for GRU models too (export_onnx.py:57)")
    sd = {k: v.detach().to(device="cpu", dtype=torch.float32) for k, v in model.state_dict().items()
          if not k.endswith("num_batches_tracked")}
    g = _Graph()
    x = "input"
    if model.global_cmvn is not None:                                              # cmvn.py:45-47
        x = g.node("Sub", [x, g.const(sd["global_cmvn.mean"], "mean")])
        if model.global_cmvn.norm_var:
            x = g.node("Mul", [x, g.const(sd["global_cmvn.istd"], "istd")])
    if kind == "fsmn":
        cache_shape = [1, bb.proj_dim, bb.cache_len, bb.fsmn_layers]
        y, r_cache = _fsmn(g, sd, bb, x, "cache")
    else:
        cache_shape = [1, model.hdim, bb.padding]
        x = g.node("Relu", [g.linear(x, sd["preprocessing.out.0.weight"], sd["preprocessing.out.0.bias"])])
        x = g.node("Transpose", [x], [_attr_ints("perm", [0, 2, 1])])
        y, r_cache = (_mdtc if kind == "mdtc" else _tcn)(g, sd, bb, x, "cache", model.hdim)
        y = g.node("Transpose", [y], [_attr_ints("perm", [0, 2, 1])])
        y = g.linear(y, sd["classifier.linear.weight"], sd["classifier.linear.bias"])   # classifier.py:63-67
    if isinstance(model.activation, torch.nn.Sigmoid):
        y = g.node("Sigmoid", [y])
    if softmax:
        y = g.node("Softmax", [y], [_attr_int("axis", 2)])                          # kws_model.py:88
    g.node("Identity", [y], out="output")
    g.node("Identity", [r_cache], out="r_cache")

    graph = b"".join(_f_bytes(1, n) for n in g.nodes) + _f_str(2, "wekws_b200")
    graph += b"".join(_f_bytes(5, t) for t in g.inits)
    graph += _f_bytes(11, _value_info("input", [1, "T", model.idim])) + _f_bytes(11, _value_info("cache", cache_shape))
    graph += _f_bytes(12, _value_info("output", [1, "T", model.odim])) + _f_bytes(12, _value_info("r_cache", cache_shape))
    meta = {"cache_dim": str(bb.proj_dim if kind == "fsmn" else model.hdim),
            "cache_len": str(bb.cache_len if kind == "fsmn" else bb.padding)}
    # ModelProto: ir_version = 1, producer_name = 2, producer_version = 3, graph = 7, opset_import = 8, metadata_props = 14
    m = _f_varint(1, IR_VERSION) + _f_str(2, "wekws_b200") + _f_str(3, "2")
    m += _f_bytes(7, graph) + _f_bytes(8, _f_str(1, "") + _f_varint(2, OPSET))
    for k, v in meta.items():
        m += _f_bytes(14, _f_str(1, k) + _f_str(2, v))
    with open(path, "wb") as f:
        f.write(m)
    return {"nodes": len(g.nodes), "initializers": len(g.inits), **meta}
