"""The FSMN kernel (fsmn.cu) at the batch sizes and chunk heights that select its other tile schedules, at the widths
of its shared-memory limit, and its training twin against it.

fsmn_launch puts S = min(64 / T, B) whole streams in each 64-row tile, so B streams make n_tiles = ceil(B / S) tiles,
the last one holding B - (n_tiles - 1) S streams and 64 - S T rows of every tile dead; the grid is min(n_tiles, SMs)
and each CTA walks its tiles with one weight ring.  wekws_model_forward cuts a call of T > 64 frames into ceil(T / 64)
equal chunks, each reading the cache the previous one wrote, and a chunk shorter than the cache (left_order - 1 +
right_order columns) takes part of its new cache from the old one.

Without a GPU: `schedule` restates that partition from the constants it reads out of fsmn.cu, and a test checks that
the GPU shapes reach every class in REQUIRED for 132 and 114 SMs; the 226 KB boundary packs, one column past it is
refused.  On the GPU every stream's output and returned cache is compared with the float64 oracle on its own, so a
tile-indexing error cannot hide behind a batch maximum; a stream's results are bit-identical whatever tile, slot or
chunking it runs in; and the training forward's kernel (fsmn_train_kernel) gives the eval kernel's bits.  `-s` prints
each case's error next to its gate.
"""
import os
import re

import pytest
import torch

from oracle import kws_head_oracle as HO
from tests.test_batch_schedules import _cdiv
from tests.test_config_sweep import (ROW_IDS, TOL_FP32, _ROW, build_config, build_row, cache_shape, inputs, kind,
                                     row_config)
from wekws_b200 import init_model, model_config, synth

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "wekws_b200", "csrc")


# ----------------------------------------------------------------------------------------------- the schedule
_CONSTS = None


def kernel_constants():
    """The tile height, GEMM pass width, ring chunk and shared-memory limit of fsmn.cu, read from its source."""
    global _CONSTS
    if _CONSTS is None:
        with open(os.path.join(CSRC, "fsmn.cu")) as f:
            src = f.read()

        def one(pattern):
            m = re.search(pattern, src)
            assert m, f"pattern not found in fsmn.cu: {pattern}"
            return int(m.group(1))
        _CONSTS = dict(ROWS=one(r"constexpr int ROWS = (\d+);"), NPASS=one(r"constexpr int NPASS = (\d+);"),
                       KC=one(r"constexpr int KC = (\d+);"),
                       SMEM=one(r"WEKWS_REQUIRE\(smem <= (\d+) \* 1024,") * 1024)
    return _CONSTS


def smem_bytes(idim, A1, D, P, A2):
    """pack_fsmn's row strides and fsmn_smem_bytes: three 64-row activation buffers and a two-slot weight ring."""
    K = kernel_constants()

    def stride(n):
        return (n + 3) // 4 * 4 + 4
    return 4 * (K["ROWS"] * (stride(max(idim, D)) + stride(max(A1, P, A2)) + stride(P)) + 2 * K["KC"] * K["NPASS"])


def schedule(B, T):
    """The launches of one forward call of B streams x T frames: per host chunk its height, streams per tile, tiles
    and streams in the last tile."""
    rows = kernel_constants()["ROWS"]
    Tc = _cdiv(T, _cdiv(T, rows))
    out = []
    for t0 in range(0, T, Tc):
        Tk = min(Tc, T - t0)
        S = min(rows // Tk, B)
        n = _cdiv(B, S)
        out.append(dict(T=Tk, S=S, tiles=n, tail=B - (n - 1) * S))
    return out


def classes(B, T, pad, sms):
    """The schedule classes one call reaches on `sms` SMs with a cache of `pad` columns."""
    ch = schedule(B, T)
    out = {f"{min(len(ch), 3)}{'+' if len(ch) >= 3 else ''} chunk{'s' if len(ch) > 1 else ''}"}
    for c in ch:
        out.add("one stream per tile" if c["S"] == 1 else "several streams per tile")
        if c["tail"] < c["S"]:
            out.add("a tail tile with fewer streams")
        if c["tiles"] > 2 * sms:
            out.add("more than two tiles per CTA")
        if c["S"] * c["T"] < kernel_constants()["ROWS"]:
            out.add("dead rows in every tile")
        if c["T"] < pad:
            out.add("a chunk shorter than the cache")
    return out


REQUIRED = {"1 chunk", "2 chunks", "3+ chunks", "one stream per tile", "several streams per tile",
            "a tail tile with fewer streams", "more than two tiles per CTA", "dead rows in every tile",
            "a chunk shorter than the cache"}

# (T, B): 64, 9, 3 and 1 streams per tile, 266 .. 300 tiles, tails of 40, 7 and 2 streams; then 2 and 3 host chunks
SHAPES = [(1, 17000), (7, 2401), (21, 800), (64, 300), (65, 300), (129, 200)]
# the shipped widths and a small row with a 31-column cache
MODELS = ["shipped", "fsmn_l20_r12"]
SHIPPED = ("fsmn", dict(input_dim=400, output_dim=2599))

# input 400, widths 140 / 250 / 180 / 184 (input_affine / linear / proj / output_affine), output 2599: 226 KB exactly
EDGE = dict(input_dim=400, output_dim=2599, input_affine_dim=140, linear_dim=250, proj_dim=180, output_affine_dim=184)


def _edge_config(A2=184):
    cfg = model_config("fsmn", input_dim=EDGE["input_dim"], output_dim=EDGE["output_dim"], activation="identity")
    cfg["backbone"].update({k: v for k, v in EDGE.items() if k not in ("input_dim", "output_dim")},
                           output_affine_dim=A2)
    return cfg


def _pad(cfg):
    return cache_shape(cfg, 1)[2]


def _model_config(model):
    """The config of a model of MODELS (no weights built)."""
    if model == "shipped":
        return model_config(SHIPPED[0], activation="identity", **SHIPPED[1])
    cfg, cleanup = row_config(model)
    cleanup()
    return cfg


# ----------------------------------------------------------------------------------------------------------- CPU
def test_schedule_constants_are_read_from_the_sources():
    K = kernel_constants()
    assert K["ROWS"] == 64 and K["SMEM"] == 226 * 1024
    assert [(c["T"], c["S"], c["tiles"], c["tail"]) for c in schedule(300, 65)] == [(33, 1, 300, 1), (32, 2, 150, 2)]
    assert [c["T"] for c in schedule(4, 129)] == [43, 43, 43]


@pytest.mark.parametrize("T,B,S,tiles,tail", [(1, 17000, 64, 266, 40), (7, 2401, 9, 267, 7), (21, 800, 3, 267, 2),
                                              (64, 300, 1, 300, 1)])
def test_schedule_of_the_single_chunk_shapes(T, B, S, tiles, tail):
    assert schedule(B, T) == [dict(T=T, S=S, tiles=tiles, tail=tail)]


@pytest.mark.parametrize("sms", [132, 114])
def test_gpu_shapes_reach_every_schedule_class(sms):
    """The GPU shapes, mapped through the schedule, reach every class in REQUIRED for each model they run (H100 SXM:
    132 SMs, PCIe: 114)."""
    for model in MODELS:
        pad = _pad(_model_config(model))
        reached = set()
        for T, B in SHAPES:
            reached |= classes(B, T, pad, sms)
        assert not REQUIRED - reached, (model, sorted(REQUIRED - reached))


def test_the_widest_model_packs_at_exactly_226_kb(native):
    """Widths that need every byte of the kernel's shared-memory limit pack; one more output_affine column (one more
    4-float stride step) needs 1 KB more and the pack refuses it, naming shared memory, before any device work."""
    assert smem_bytes(400, 140, 250, 180, 184) == kernel_constants()["SMEM"] == 231424
    assert smem_bytes(400, 140, 250, 180, 185) == 232448
    m = synth.randomize_(init_model(_edge_config())).eval()
    m._build_handle(finalize=False)
    m._release()
    m = synth.randomize_(init_model(_edge_config(A2=185))).eval()
    with pytest.raises(RuntimeError, match="wekws_model_pack.*shared memory"):
        m._build_handle(finalize=False)
    m._release()


# ----------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda:0"
_SLICE = 1 << 24            # oracle elements per slice of streams


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(model):
        if model not in cache:
            if model == "shipped":
                cfg, m = build_config(*SHIPPED, init_model)
            elif model == "edge":
                cfg = _edge_config()
                m = synth.randomize_(init_model(cfg)).eval()
            else:
                cfg, m = build_row(model, init_model)
            # the float64 oracle runs on the device: 17000 streams of the shipped widths are slow on the host
            sd = {k: v.detach().to(DEV, torch.float64) for k, v in m.state_dict().items()}
            cache[model] = (cfg, m.to(DEV), sd)
        return cache[model]
    yield get
    cache.clear()


def _per_stream(got, ref):
    """(max |got - ref|, max |ref|) of each stream (dimension 0)."""
    d = (got.to(ref.dtype) - ref).abs().flatten(1).amax(1)
    return d, ref.abs().flatten(1).amax(1)


def compare_streams(what, cfg, sd, x, cache, y, c):
    """Every stream's output and returned cache against the float64 oracle, each under its own gate TOL_FP32 x
    max(1, max |ref| of that stream)."""
    B, T = x.shape[:2]
    per = T * cfg["output_dim"] + 2 * cache[0].numel()
    step = max(1, _SLICE // per)
    worst = dict(out=0.0, cache=0.0)
    for s0 in range(0, B, step):
        s = slice(s0, min(B, s0 + step))
        y_ref, c_ref = HO.kws_forward(sd, cfg, x[s].to(DEV, torch.float64), cache[s].to(DEV, torch.float64))
        for name, got, ref in (("out", y[s], y_ref), ("cache", c[s], c_ref)):
            err, mag = _per_stream(got, ref)
            ratio = err / (TOL_FP32 * mag.clamp(min=1.0))
            worst[name] = max(worst[name], float(ratio.max()))
            bad = torch.nonzero(ratio > 1).flatten()
            assert bad.numel() == 0, (what, name, [s0 + int(b) for b in bad[:8]], float(err[bad[0]]))
    print(f"{what}: largest error / gate of one stream: out {worst['out']:.3f}, cache {worst['cache']:.3f}")
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("T,B", SHAPES)
@pytest.mark.parametrize("model", MODELS)
def test_gpu_every_stream_matches_float64_oracle(model, T, B, models):
    """Every stream against the float64 oracle, from a random cache, at the shapes that reach each schedule class."""
    cfg, m, sd = models(model)
    x, cache = inputs(cfg, B, T, seed=11 * B + T)
    y, c = m(x.to(DEV), cache.to(DEV))
    assert tuple(c.shape) == cache_shape(cfg, B)
    compare_streams(f"{model} T={T} B={B}", cfg, sd, x, cache, y, c)


@pytest.mark.gpu
@pytest.mark.parametrize("model", MODELS)
def test_gpu_results_depend_only_on_the_stream(model, models):
    """A frame's output and the returned cache depend, bit for bit, only on that stream's features and cache: every
    row runs the same FMA sequence whatever tile, stream slot or chunk it lands in, and cache columns are exact copies
    of projections.  So a stream alone equals its row of a 2401-stream call, streamed chunks of 1, 7, 33, 64 and 65
    frames (some shorter than the cache) equal one call, and permuting the streams permutes the results."""
    cfg, m, _ = models(model)
    B, T = 2401, 7
    x, cache = inputs(cfg, B, T, seed=21)
    xd, cd = x.to(DEV), cache.to(DEV)
    y, c = m(xd, cd)
    for b in (0, 8, 9, 1000, 2399, 2400):       # the first and last slot of a 9-stream tile, the 7-stream tail tile
        y1, c1 = m(xd[b:b + 1].contiguous(), cd[b:b + 1].contiguous())
        assert torch.equal(y1[0], y[b]) and torch.equal(c1[0], c[b]), (model, b)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(3)).to(DEV)
    yp, cp = m(xd[perm].contiguous(), cd[perm].contiguous())
    assert torch.equal(yp, y[perm]) and torch.equal(cp, c[perm]), model

    chunks = [1, 7, 33, 64, 65]
    B = 300
    x, cache = inputs(cfg, B, sum(chunks), seed=22)
    xd, cd = x.to(DEV), cache.to(DEV)
    y_full, c_full = m(xd, cd)
    ys, c, t0 = [], cd, 0
    for n in chunks:
        y, c = m(xd[:, t0:t0 + n].contiguous(), c)
        ys.append(y)
        t0 += n
    assert any(n < _pad(cfg) for n in chunks)
    assert torch.equal(torch.cat(ys, 1), y_full) and torch.equal(c, c_full), model


@pytest.mark.gpu
def test_gpu_widest_model_matches_oracle_and_trains_bit_exact(models):
    """The 226 KB model at 300 streams x 40 frames (one stream per tile, 300 tiles): every stream against the float64
    oracle, and the training-mode forward (fsmn_train_kernel) gives the eval kernel's bits."""
    cfg, m, sd = models("edge")
    B, T = 300, 40
    x, cache = inputs(cfg, B, T, seed=40)
    xd = x.to(DEV)
    y, c = m(xd, cache.to(DEV))
    compare_streams("edge T=40 B=300", cfg, sd, x, cache, y, c)
    _assert_training_forward_is_eval(m, xd)


def _assert_training_forward_is_eval(m, xd):
    with torch.no_grad():
        y_eval, c_eval = m.eval()(xd)
    try:
        m.train()
        y, c = m(xd)
        assert y.requires_grad
    finally:
        m.eval()
    assert torch.equal(y.detach().view(torch.int32), y_eval.view(torch.int32))
    assert torch.equal(c.view(torch.int32), c_eval.view(torch.int32))


_TRAINABLE = [r for r in ROW_IDS if kind(r) == "fsmn" and "activation" not in _ROW[r][2]
              and _ROW[r][2].get("left_order", 10) + _ROW[r][2].get("right_order", 2) <= 32]


@pytest.mark.gpu
@pytest.mark.parametrize("row", _TRAINABLE)
def test_gpu_training_forward_equals_eval_for_every_sweep_row(row, models):
    """fsmn_train_kernel against fsmn_kernel at every trainable FSMN configuration of the sweep: 37 streams of 129
    frames (three host chunks, each storing its activations), logits and cache bit for bit."""
    cfg, m, _ = models(row)
    x, _ = inputs(cfg, 37, 129, seed=129)
    _assert_training_forward_is_eval(m, x.to(DEV))
