"""Every backbone kernel across the model configurations it accepts, not only the shipped recipe shapes.

ROWS below lists about fifty configurations.  Each sits on a kernel variant no recipe reaches (one A atom, 17 MDTC
blocks, generic DS-TCN cache pitch, one-layer GRU, ...) or one step past an eligibility edge, and names the kernel a
large-batch call with T >= 8 takes:

    Mdtc / Tcn / DsTcn    the tensor-core kernel of that backbone (mdtc_tc.cu, tcn_tc.cu, dstcn_tc.cu)
    DsTcn+linear_tc       the DS-TCN kernel with the classifier as its own tensor-core GEMM (output_dim > 4)
    Gru                   the tensor-core GRU (batch thresholds under "auto", always under "tensor")
    fp32                  the FP32 kernels only (conv_backbone.cu, gru.cu)
    Fsmn                  the fused FP32 FSMN kernel (fsmn.cu), the only one that model has

Without a GPU: the kernel choice (a tensor-core model packs a weight image), the packed FP32 weights against the oracle,
and the oracle against the reference (live when its sources are present, else tests/golden/config_sweep.npz, made by
oracle/make_sweep_golden.py).  On the GPU every row runs under each precision mode against the float64 oracle at
shapes that cross the chosen kernel's chunk height, with a random cache; plus streaming, batch-size, misaligned-input
and in-place-cache properties.  `-s` prints the measured error of each case next to its gate.
"""
import contextlib
import io
import os

import pytest
import torch

from oracle import kws_head_oracle as HO
from oracle import kws_oracle as O
from tests import packed_eval as PE
from tests.conftest import golden, have_reference, reference_init_model
from wekws_b200 import init_model, synth
from wekws_b200.configs import model_config

# (id, recipe, overrides, kernel).  Overrides: model_config arguments (input_dim, output_dim, activation, cmvn,
# norm_var), backbone fields (num_stack, stack_size, kernel_size, num_layers and FSMN_FIELDS), hidden_dim, head
# ("global" / "last").  Hidden 64 for MDTC and TCN, 256 for DS-TCN, 128 for GRU unless given; output_dim 1 unless given.
# The rows output logits (activation identity) unless they ask for the sigmoid: a saturated sigmoid would hide
# differences the gates must see.
FSMN_FIELDS = ("input_affine_dim", "linear_dim", "proj_dim", "output_affine_dim", "left_order", "right_order",
               "left_stride", "right_stride")
FSMN_SMALL = dict(input_dim=40, output_dim=7, input_affine_dim=24, linear_dim=36, proj_dim=16, output_affine_dim=20,
                  num_layers=3, left_order=10, right_order=2)
ROWS = [
    # MDTC tensor-core kernel: kernel 5, stack_size <= 4, <= 17 blocks, input_dim % 8 == 0 and <= 96, output_dim <= 8
    ("mdtc_1x1_i40_o3", "mdtc", dict(num_stack=1, stack_size=1, input_dim=40, output_dim=3, activation="sigmoid"),
     "Mdtc"),
    ("mdtc_2x3_i96_o8", "mdtc", dict(num_stack=2, stack_size=3, input_dim=96, output_dim=8), "Mdtc"),
    ("mdtc_8x2_i64", "mdtc", dict(num_stack=8, stack_size=2, input_dim=64), "Mdtc"),
    ("mdtc_2x3_i40_last", "mdtc", dict(num_stack=2, stack_size=3, input_dim=40, output_dim=4, head="last"), "Mdtc"),
    ("mdtc_6x3", "mdtc", dict(num_stack=6, stack_size=3), "fp32"),                          # 19 blocks
    ("mdtc_4x4_o9", "mdtc", dict(output_dim=9), "fp32"),
    ("mdtc_k3", "mdtc", dict(kernel_size=3), "fp32"),                                       # pads 2 .. 16
    ("mdtc_k7", "mdtc", dict(kernel_size=7), "fp32"),                                       # pads 6 .. 48
    ("mdtc_2x5", "mdtc", dict(num_stack=2, stack_size=5), "fp32"),                          # padmax 64
    ("mdtc_i13_cmvn", "mdtc", dict(input_dim=13, cmvn=True), "fp32"),
    ("mdtc_h128_2x3", "mdtc", dict(hidden_dim=128, num_stack=2, stack_size=3), "fp32"),
    ("mdtc_h256_1x2", "mdtc", dict(hidden_dim=256, num_stack=1, stack_size=2), "fp32"),
    # dense TCN tensor-core kernel: hidden 64, input_dim % 8 == 0, output_dim <= 8, roundup4(padmax) + 8 <= 504
    ("tcn_k3x5_i40_o8", "tcn", dict(kernel_size=3, num_layers=5, input_dim=40, output_dim=8, activation="sigmoid"),
     "Tcn"),
    ("tcn_k2x3", "tcn", dict(kernel_size=2, num_layers=3), "Tcn"),
    ("tcn_k8x7", "tcn", dict(kernel_size=8, num_layers=7), "Tcn"),                         # padmax 448: 56-frame chunks
    ("tcn_k4x8", "tcn", dict(kernel_size=4, num_layers=8), "Tcn"),                         # padmax 384: 120 frames
    ("tcn_k8x4_o9", "tcn", dict(output_dim=9), "fp32"),
    ("tcn_k5x8", "tcn", dict(kernel_size=5, num_layers=8), "fp32"),                        # padmax 512
    ("tcn_h128", "tcn", dict(hidden_dim=128), "fp32"),
    ("tcn_h32", "tcn", dict(hidden_dim=32), "fp32"),
    ("tcn_i13", "tcn", dict(input_dim=13), "fp32"),
    # DS-TCN tensor-core kernel: hidden 256, kernel 8, input_dim % 8 == 0; output_dim > 4 adds the linear_tc GEMM
    ("dstcn_1l", "ds_tcn", dict(num_layers=1), "DsTcn"),                                   # cache pitch 7
    ("dstcn_3l_i40_o4", "ds_tcn", dict(num_layers=3, input_dim=40, output_dim=4), "DsTcn"),
    ("dstcn_5l_o5", "ds_tcn", dict(num_layers=5, output_dim=5, activation="sigmoid"), "DsTcn+linear_tc"),
    ("dstcn_4l_o128", "ds_tcn", dict(output_dim=128), "DsTcn+linear_tc"),
    ("dstcn_4l_o129", "ds_tcn", dict(output_dim=129), "DsTcn+linear_tc"),
    ("dstcn_k3", "ds_tcn", dict(kernel_size=3), "fp32"),
    ("dstcn_h128", "ds_tcn", dict(hidden_dim=128), "fp32"),
    ("dstcn_i13", "ds_tcn", dict(input_dim=13), "fp32"),
    ("dstcn_global_o11", "ds_tcn", dict(output_dim=11, head="global"), "fp32"),           # pool epilogue, hidden 256
    ("dstcn_last_o11", "ds_tcn", dict(output_dim=11, head="last"), "fp32"),
    # GRU tensor-core kernel: hidden 128, 1 or 2 layers, input_dim <= 96
    ("gru_1l_i40", "gru", dict(num_layers=1, input_dim=40, activation="sigmoid"), "Gru"),
    ("gru_i96", "gru", dict(input_dim=96), "Gru"),
    ("gru_i13", "gru", dict(input_dim=13), "Gru"),                                         # scalar feature load
    ("gru_i1", "gru", dict(input_dim=1), "Gru"),
    ("gru_3l", "gru", dict(num_layers=3), "fp32"),
    ("gru_4l", "gru", dict(num_layers=4), "fp32"),
    ("gru_i97", "gru", dict(input_dim=97), "fp32"),
    # FSMN kernel (fsmn.cu, FP32 only): widths input_affine / linear / proj / output_affine 24 / 36 / 16 / 20, 3 layers,
    # orders 10 / 2, input 40, output 7 unless given (FSMN_SMALL); cache (B, proj, left_order - 1 + right_order, layers)
    ("fsmn_l1_r1", "fsmn", dict(FSMN_SMALL, left_order=1, right_order=1, num_layers=1), "Fsmn"),     # cache of 1
    ("fsmn_l1_r5", "fsmn", dict(FSMN_SMALL, left_order=1, right_order=5), "Fsmn"),                  # right taps only
    ("fsmn_l20_r12", "fsmn", dict(FSMN_SMALL, left_order=20, right_order=12), "Fsmn"),  # 32 taps: the backward's limit
    ("fsmn_l60_r20", "fsmn", dict(FSMN_SMALL, left_order=60, right_order=20), "Fsmn"),  # cache of 79 > a 64-row tile
    ("fsmn_odd_cmvn", "fsmn", dict(FSMN_SMALL, input_dim=13, input_affine_dim=7, linear_dim=33, proj_dim=5,
                                   output_affine_dim=9, output_dim=1, cmvn=True, norm_var=False), "Fsmn"),  # K tails 1, 3
    ("fsmn_wide", "fsmn", dict(FSMN_SMALL, input_dim=80, input_affine_dim=129, linear_dim=257, proj_dim=129,
                               output_affine_dim=129, output_dim=129), "Fsmn"),              # two 128-column passes
    ("fsmn_16l", "fsmn", dict(FSMN_SMALL, num_layers=16), "Fsmn"),                          # the pack's layer limit
    ("fsmn_sigmoid_o2", "fsmn", dict(FSMN_SMALL, output_dim=2, activation="sigmoid"), "Fsmn"),
    ("fsmn_strided", "fsmn", dict(FSMN_SMALL, left_order=4, right_order=1, left_stride=2, right_stride=3),
     "Fsmn"),                                                                  # cache 4, FSMN.padding 9
    ("fsmn_shipped", "fsmn", dict(input_dim=400, output_dim=2599), "Fsmn"),                 # fsmn_ctc.yaml
]
ROW_IDS = [r[0] for r in ROWS]
_ROW = {r[0]: r for r in ROWS}
TENSOR_CORE = ("Mdtc", "Tcn", "DsTcn", "DsTcn+linear_tc", "Gru")

# the rows the reference golden covers (oracle/make_sweep_golden.py) and its inputs
GOLDEN_ROWS = ["tcn_k3x5_i40_o8", "tcn_k8x7", "dstcn_5l_o5", "mdtc_1x1_i40_o3", "gru_1l_i40", "gru_3l", "fsmn_l1_r5",
               "fsmn_l20_r12"]
GOLDEN_B, GOLDEN_T = 2, (98, 9)      # a 1 s clip from a random cache, then 9 frames with the cache carried

# A DS-TCN with 6 layers packs, but the FP32 conv kernel every conv model keeps cannot hold one frame of it
TOO_DEEP_DSTCN = ("ds_tcn", dict(num_layers=6))

TOL_TC, TOL_FP32 = 1e-4, 2e-5        # x max(1, max |ref|)


def kind(row_id):
    return _ROW[row_id][1]


def expected(row_id):
    return _ROW[row_id][3]


def row_config(row_id):
    """-> (cfg, cleanup callable): the model config of a row (a temporary CMVN stats file if it has one)."""
    _, name, ov, _ = _ROW[row_id]
    return _config(name, ov)


def _config(name, ov):
    ov = dict(ov)
    ov.setdefault("activation", "identity")
    bb_keys = {k: ov.pop(k) for k in ("num_stack", "stack_size", "kernel_size", "num_layers") + FSMN_FIELDS if k in ov}
    hidden, head = ov.pop("hidden_dim", None), ov.pop("head", None)
    cmvn_file = synth.write_cmvn_json(ov.get("input_dim", 80)) if ov.pop("cmvn", False) else None
    cfg = model_config(name, cmvn_file=cmvn_file, **ov)
    cfg["backbone"].update(bb_keys)
    if name == "fsmn" and ov["activation"] == "sigmoid":
        # the config grammar gives an FSMN model (classifier 'identity') the Identity activation only: build_config
        # sets the Sigmoid module, and the oracle reads the missing key as the Sigmoid
        del cfg["activation"]
    if hidden is not None:
        cfg["hidden_dim"] = hidden
        if name.startswith("mdtc"):
            cfg["backbone"]["hidden_dim"] = hidden
    if head is not None:
        cfg["classifier"] = dict(type=head, dropout=0.5)
    return cfg, (lambda: os.unlink(cmvn_file)) if cmvn_file else (lambda: None)


def build_row(row_id, factory, seed=777):
    """-> (cfg, model): `factory` (the reference's or this package's init_model) with the synthetic weights."""
    _, name, ov, _ = _ROW[row_id]
    return build_config(name, ov, factory, seed)


def build_config(name, ov, factory, seed=777):
    """build_row for a recipe config `name` with the overrides `ov` of a ROWS entry ({} for the shipped shape)."""
    cfg, cleanup = _config(name, ov)
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            torch.manual_seed(seed)
            model = factory(cfg)
    finally:
        cleanup()
    if cfg["backbone"]["type"] == "fsmn" and "activation" not in cfg:
        model.activation = torch.nn.Sigmoid()
    synth.randomize_(model, seed=seed)
    model.eval()
    return cfg, model


def cache_shape(cfg, B):
    bb = cfg["backbone"]
    if bb["type"] == "gru":
        return (bb["num_layers"], B, cfg["hidden_dim"])
    if bb["type"] == "fsmn":              # the blocks run with strides 1 whatever the config says: no FSMN.padding
        return (B, bb["proj_dim"], bb["left_order"] - 1 + bb["right_order"], bb["num_layers"])
    return (B, cfg["hidden_dim"], O.backbone_padding(cfg))


def inputs(cfg, B, T, seed):
    """Features (log-mel-like when the model has a CMVN) and a 0.5 N(0, 1) cache."""
    x = synth.features(B, T, cfg["input_dim"], seed=seed, cmvn_like="cmvn" in cfg)
    cache = 0.5 * torch.randn(*cache_shape(cfg, B), generator=torch.Generator().manual_seed(seed + 1))
    return x, cache


def golden_inputs(cfg):
    """The golden file's inputs, regenerated from their seeds: two feature chunks and the first call's cache."""
    x0, cache = inputs(cfg, GOLDEN_B, GOLDEN_T[0], seed=600)
    x1, _ = inputs(cfg, GOLDEN_B, GOLDEN_T[1], seed=602)
    return x0, cache, x1


def _sd(model, dtype=torch.float32):
    return {k: (v.detach().to("cpu", dtype) if v.dtype.is_floating_point else v.detach().cpu())
            for k, v in model.state_dict().items()}


def _scaled_err(got, ref):
    return float((got.double() - ref.double()).abs().max()) / max(1.0, float(ref.abs().max()))


# ----------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("row", ROW_IDS)
def test_kernel_choice_is_pinned_by_the_pack(row, native):
    """A model gets a tensor-core weight image exactly when its row expects a tensor-core kernel."""
    _, m = build_row(row, init_model)
    h = m._build_handle(finalize=False)
    try:
        has_image = native.lib().wekws_model_packed_floats(h, 2) > 0
    finally:
        m._release()
    assert has_image == (expected(row) in TENSOR_CORE), (row, expected(row))


@pytest.mark.parametrize("row", [r for r in ROW_IDS if "head" not in _ROW[r][2] and kind(r) != "fsmn"])
def test_fold_and_pack_reproduce_the_oracle(row, native):
    """The packed FP32 weight stream (BN folded, every kernel's source), evaluated with plain torch ops, against the
    oracle with a random cache."""
    cfg, m = build_row(row, init_model)
    sd = _sd(m)
    h = m._build_handle(finalize=False)
    try:
        stream, vec = PE.read_packed(native, h)
    finally:
        m._release()
    bb = cfg["backbone"]
    has_cmvn = m.global_cmvn is not None
    sig = cfg.get("activation", {}).get("type", "sigmoid") == "sigmoid"
    x, cache = inputs(cfg, 3, 21, seed=3)
    y_ref, c_ref = HO.kws_forward(sd, cfg, x, cache)
    if bb["type"] == "gru":
        y, c = PE.eval_gru(vec, cfg["hidden_dim"], bb["num_layers"], cfg["input_dim"], cfg["output_dim"], sig,
                           has_cmvn, x, cache)
    else:
        kd = "mdtc" if bb["type"] == "mdtc" else ("ds_tcn" if bb.get("ds") else "tcn")
        dils = [1] + [2 ** l for _ in range(bb["num_stack"]) for l in range(bb["stack_size"])] \
            if kd == "mdtc" else [2 ** i for i in range(bb["num_layers"])]
        y, c = PE.eval_conv(stream, vec, kd, m.hdim, cfg["input_dim"], cfg["output_dim"], bb.get("kernel_size", 8),
                            dils, bb.get("stack_size", 1), sig, has_cmvn, x, cache)
    assert _scaled_err(y, y_ref) <= 2e-5, row
    assert _scaled_err(c, c_ref) <= 2e-5, row


@pytest.mark.parametrize("row", ROW_IDS)
def test_random_cache_moves_the_output_far_beyond_the_gate(row):
    """A kernel that ignored its cache (or read the wrong halo) must fail the GPU comparisons: at the shapes they use,
    the float64 oracle's output with the random cache is more than 50x the loosest gate away from the zero-cache one."""
    cfg, m = build_row(row, init_model)
    sd = _sd(m, torch.float64)
    # a `last` head reads one frame, 40 frames past the cache: there the cache is pinned by the returned cache only
    for B, T in ((1, 8),) if m.head == "last" else ((1, 8), (2, 40)):
        x, cache = inputs(cfg, B, T, seed=11)
        y, _ = HO.kws_forward(sd, cfg, x.double(), cache.double())
        y0, _ = HO.kws_forward(sd, cfg, x.double(), torch.zeros_like(cache, dtype=torch.float64))
        assert _scaled_err(y0, y) > 50 * TOL_TC, (row, B, T, _scaled_err(y0, y))


@pytest.mark.parametrize("row", GOLDEN_ROWS)
def test_oracle_matches_reference_sweep_golden(row):
    """The oracle against the outputs the real reference produced for these rows (oracle/make_sweep_golden.py)."""
    g = golden("config_sweep")
    cfg, m = build_row(row, init_model)
    assert abs(synth.state_digest(m) - float(g[row + "/digest"])) < 1e-6 * float(g[row + "/digest"])
    x0, cache, x1 = golden_inputs(cfg)
    for name, t in (("x0", x0), ("cache", cache), ("x1", x1)):
        want = float(g[f"{row}/{name}_abs_sum"])
        assert abs(float(t.double().abs().sum()) - want) < 1e-9 * want, (row, name)
    sd = _sd(m)
    y0, c = HO.kws_forward(sd, cfg, x0, cache)
    y1, c = HO.kws_forward(sd, cfg, x1, c)
    assert _scaled_err(y0, torch.from_numpy(g[row + "/y0"])) <= 2e-6, row
    assert _scaled_err(y1, torch.from_numpy(g[row + "/y1"])) <= 2e-6, row
    assert _scaled_err(c[..., -16:], torch.from_numpy(g[row + "/c1_tail"])) <= 2e-6, row


@pytest.mark.skipif(not have_reference(), reason="reference sources not present")
@pytest.mark.parametrize("row", ROW_IDS)
def test_oracle_matches_live_reference(row):
    """The oracle against the reference's own modules at every row, three calls with the cache carried."""
    cfg, ref = build_row(row, reference_init_model())
    sd = ref.state_dict()
    gru = cfg["backbone"]["type"] == "gru"
    x, c_ref = inputs(cfg, 2, 23, seed=5)
    c_or = c_ref
    with torch.no_grad():
        for i in range(3):
            y_ref, c_ref = ref(x, c_ref)
            y_or, c_or = HO.kws_forward(sd, cfg, x, c_or)
            assert _scaled_err(y_or, y_ref) <= 2e-6, (row, i)
            assert (c_ref - c_or).abs().max() <= 1e-5, (row, i)
            if not gru and i == 0:
                c_ref = c_or = torch.zeros(0, 0, 0)          # start of stream: the reference's empty cache


def test_a_too_deep_ds_tcn_is_refused_when_it_is_finalized(native):
    """A 6-layer DS-TCN (widest cache slice 224 frames) packs, and the tensor-core kernel would not need the FP32 tile;
    but the FP32 conv kernel every conv model keeps for T < 8 cannot hold one frame of it, so finalize refuses it
    before it touches the device, naming the cause."""
    name, ov = TOO_DEEP_DSTCN
    cfg, cleanup = _config(name, ov)
    cleanup()
    m = synth.randomize_(init_model(cfg)).eval()
    m._build_handle(finalize=False)                           # the pack itself succeeds
    with pytest.raises(RuntimeError, match="wekws_model_finalize.*shared memory.*224"):
        m._build_handle(finalize=True)
    m._release()


# ----------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda:0"
_BOLD_T = [1, 7, 8, 40, 56, 57, 98, 120, 121, 125, 128, 250]   # around the 56- and 120-frame chunks of padmax 448 / 384


def _times(row):
    if row in ("tcn_k8x7", "tcn_k4x8"):
        return _BOLD_T
    if expected(row) == "Fsmn":        # 64-row tiles: 1 .. 64 streams per tile, then 2 and 3 host chunks (33 + 32, 3 x 43)
        return [1, 7, 8, 21, 33, 40, 63, 64, 65, 129]
    extra = {"Mdtc": [129, 257], "Tcn": [129, 257], "DsTcn": [121], "DsTcn+linear_tc": [121], "Gru": [129],
             "fp32": [300]}[expected(row)]
    return [1, 7, 8, 40] + extra


def _precisions(row):
    return ["auto", "fp32", "tensor"] if kind(row) == "gru" else ["auto", "fp32"]


_SHAPES = [(row, B, T) for row in ROW_IDS for B in (1, 37) for T in _times(row)]


@pytest.fixture(scope="module")
def sweep_models():
    cache = {}

    def get(row):
        if row not in cache:
            cfg, m = build_row(row, init_model)
            cache[row] = (cfg, m.to(DEV), _sd(m, torch.float64))
        return cache[row]
    yield get
    cache.clear()


def _takes_tensor_cores(row, m, B, T):
    """The answer the table gives for a call of B x T under the model's precision mode."""
    if m.precision == "fp32" or expected(row) not in TENSOR_CORE:
        return False
    if kind(row) == "gru":
        return m.precision == "tensor" or B >= (640 if T == 1 else 400 if T < 8 else 256)
    return T >= 8


def _gate(tc, ref):
    return (TOL_TC if tc else TOL_FP32) * max(1.0, float(ref.abs().max()))


def _check(what, tc, y, c, y_ref, c_ref):
    ey = float((y.cpu().double() - y_ref).abs().max())
    ec = float((c.cpu().double() - c_ref).abs().max())
    gy, gc = _gate(tc, y_ref), _gate(tc, c_ref)
    print(f"{what} {'tensor-core' if tc else 'fp32'}: out {ey:.2e} (gate {gy:.1e}), cache {ec:.2e} (gate {gc:.1e})")
    assert ey <= gy and ec <= gc, (what, ey, gy, ec, gc)


@pytest.mark.gpu
@pytest.mark.parametrize("row,B,T", _SHAPES)
def test_gpu_matches_float64_oracle(row, B, T, sweep_models):
    """Every precision mode against the float64 oracle, output and returned cache, from a random cache; the kernel
    taken is the one the table names."""
    cfg, m, sd64 = sweep_models(row)
    x, cache = inputs(cfg, B, T, seed=1000 * B + T)
    y_ref, c_ref = HO.kws_forward(sd64, cfg, x.double(), cache.double())
    xd, cd = x.to(DEV), cache.to(DEV)
    try:
        for prec in _precisions(row):
            m.precision = prec
            y, c = m(xd, cd)
            tc = _takes_tensor_cores(row, m, B, T)
            assert m.uses_tensor_cores(T, B) == tc, (row, prec, B, T)
            if prec == "auto" and kind(row) != "gru":
                assert m.uses_tensor_cores(T) == (T >= 8 and expected(row) in TENSOR_CORE)
            _check(f"{row} B={B} T={T} {prec}", tc, y, c, y_ref, c_ref)
    finally:
        m.precision = "auto"
    if kind(row) == "gru":
        assert m.uses_tensor_cores(T) == (expected(row) == "Gru")       # a large batch


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROW_IDS)
def test_gpu_b300_rows_and_stream_permutation(row, sweep_models):
    """300 streams (several passes per CTA): rows against the float64 oracle, and permuting the streams permutes the
    outputs and caches bit for bit."""
    cfg, m, sd64 = sweep_models(row)
    B, T = 300, 40
    x, cache = inputs(cfg, B, T, seed=300)
    xd, cd = x.to(DEV), cache.to(DEV)
    y, c = m(xd, cd)
    rows = [0, 1, 150, 299]
    cr = cache[:, rows] if kind(row) == "gru" else cache[rows]
    y_ref, c_ref = HO.kws_forward(sd64, cfg, x[rows].double(), cr.double())
    got_c = c[:, rows] if kind(row) == "gru" else c[rows]
    _check(f"{row} B=300 T=40 auto", _takes_tensor_cores(row, m, B, T), y[rows], got_c, y_ref, c_ref)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(0)).to(DEV)
    cp = cd[:, perm] if kind(row) == "gru" else cd[perm]
    yp, cpo = m(xd[perm].contiguous(), cp.contiguous())
    assert torch.equal(yp, y[perm])
    assert torch.equal(cpo, c[:, perm] if kind(row) == "gru" else c[perm])


@pytest.mark.gpu
@pytest.mark.parametrize("row", ROW_IDS)
def test_gpu_streaming_equals_one_call(row, sweep_models):
    """8 + 1 + 40 frames with the cache carried == one call of 49 frames (the head rows pool per call, so for them
    only the cache is compared)."""
    cfg, m, _ = sweep_models(row)
    B = 37
    x, cache = inputs(cfg, B, 49, seed=49)
    xd, cd = x.to(DEV), cache.to(DEV)
    y_full, c_full = m(xd, cd)
    c, ys = cd, []
    for t0, t1 in ((0, 8), (8, 9), (9, 49)):
        y, c = m(xd[:, t0:t1].contiguous(), c)
        ys.append(y)
    tol = 2e-5
    assert _scaled_err(c.cpu(), c_full.cpu()) <= tol, row
    if m.head is None:
        e = _scaled_err(torch.cat(ys, 1).cpu(), y_full.cpu())
        print(f"{row} streamed 8 + 1 + 40 vs one call: {e:.2e} (gate {tol:.0e})")
        assert e <= tol, row


@pytest.mark.gpu
@pytest.mark.parametrize("row", ["mdtc_1x1_i40_o3", "tcn_k3x5_i40_o8", "dstcn_3l_i40_o4"])
def test_gpu_misaligned_inputs_fall_back_to_fp32(row, sweep_models):
    """Features (and, for MDTC, the cache) 4 bytes off a 16-byte boundary: the call takes the FP32 kernel and gives
    exactly the FP32 result of aligned inputs (same kernel, same operands, same summation order)."""
    cfg, m, _ = sweep_models(row)
    B, T = 37, 40
    x, cache = inputs(cfg, B, T, seed=77)
    xd, cd = x.to(DEV), cache.to(DEV)

    def off_by_one(t):
        buf = torch.empty(t.numel() + 4, device=DEV)
        v = buf[1:1 + t.numel()].view(t.shape)
        v.copy_(t)
        assert v.is_contiguous() and v.data_ptr() % 16 == 4
        return v
    try:
        m.precision = "fp32"
        y32, c32 = m(xd, cd)
    finally:
        m.precision = "auto"
    y_tc, _ = m(xd, cd)
    assert m.uses_tensor_cores(T, B) and not torch.equal(y_tc, y32)
    y, c = m(off_by_one(xd), cd)
    assert torch.equal(y, y32) and torch.equal(c, c32)
    if kind(row) == "mdtc":
        y, c = m(xd, off_by_one(cd))
        assert torch.equal(y, y32) and torch.equal(c, c32)


@pytest.mark.gpu
@pytest.mark.parametrize("T", [40, 200])
@pytest.mark.parametrize("row", ["mdtc_1x1_i40_o3", "tcn_k3x5_i40_o8", "dstcn_3l_i40_o4", "dstcn_5l_o5",
                                 "dstcn_1l", "gru_1l_i40", "fsmn_l60_r20"])
def test_gpu_in_place_cache_through_the_c_abi(row, T, sweep_models, native):
    """wekws_model_forward with d_in_cache == d_out_cache (what the native runtime shim does) for 300 streams equals
    the call with separate buffers bit for bit."""
    cfg, m, _ = sweep_models(row)
    B = 300
    x, cache = inputs(cfg, B, T, seed=5 * T)
    xd, cd = x.to(DEV), cache.to(DEV)
    y_sep, c_sep = m(xd, cd)
    assert m.uses_tensor_cores(T, B) == (expected(row) in TENSOR_CORE)
    h = m._ensure(torch.device(DEV))
    m._apply_precision(h)
    buf = cd.clone()
    out = torch.empty_like(y_sep)
    stream = torch.cuda.current_stream(torch.device(DEV)).cuda_stream
    native.check(native.lib().wekws_model_forward(h, xd.data_ptr(), buf.data_ptr(), out.data_ptr(), buf.data_ptr(),
                                                  B, T, 0, stream), "wekws_model_forward")
    torch.cuda.synchronize()
    assert torch.equal(out, y_sep), row
    assert torch.equal(buf, c_sep), row


@pytest.mark.gpu
@pytest.mark.parametrize("row", [r for r in ROW_IDS if kind(r) != "gru" and expected(r) in TENSOR_CORE])
def test_gpu_launch_count(row, sweep_models, native):
    """A 40-frame call fits one chunk of every tensor-core conv kernel: one backbone launch, plus the classifier GEMM
    behind DS-TCN when output_dim > 4, plus the head kernel."""
    cfg, m, _ = sweep_models(row)
    x, cache = inputs(cfg, 37, 40, seed=2)
    xd, cd = x.to(DEV), cache.to(DEV)
    m(xd, cd)
    torch.cuda.synchronize()
    n0 = native.launch_count()
    m(xd, cd)
    torch.cuda.synchronize()
    want = 1 + (expected(row) == "DsTcn+linear_tc") + (m.head is not None)
    assert native.launch_count() - n0 == want, row


@pytest.mark.gpu
@pytest.mark.parametrize("row", GOLDEN_ROWS)
def test_gpu_matches_reference_sweep_golden(row, sweep_models):
    """The kernels against the real reference's outputs (tests/golden/config_sweep.npz) under each precision mode."""
    g = golden("config_sweep")
    cfg, m, _ = sweep_models(row)
    x0, cache, x1 = golden_inputs(cfg)
    try:
        for prec in _precisions(row):
            m.precision = prec
            y0, c = m(x0.to(DEV), cache.to(DEV))
            y1, c = m(x1.to(DEV), c)
            for name, y, T in (("y0", y0, GOLDEN_T[0]), ("y1", y1, GOLDEN_T[1])):
                ref = torch.from_numpy(g[f"{row}/{name}"])
                tc = _takes_tensor_cores(row, m, GOLDEN_B, T)
                e = float((y.cpu() - ref).abs().max())
                print(f"{row} {name} {prec} vs reference: {e:.2e} (gate {_gate(tc, ref):.1e})")
                assert e <= _gate(tc, ref), (row, name, prec)
            tail = torch.from_numpy(g[row + "/c1_tail"])
            assert float((c[..., -16:].cpu() - tail).abs().max()) <= _gate(True, tail), (row, prec)
    finally:
        m.precision = "auto"


@pytest.mark.gpu
def test_gpu_a_too_deep_ds_tcn_raises_on_the_first_call():
    name, ov = TOO_DEEP_DSTCN
    cfg, cleanup = _config(name, ov)
    cleanup()
    m = synth.randomize_(init_model(cfg)).eval().to(DEV)
    with pytest.raises(RuntimeError, match="wekws_model_finalize.*shared memory"):
        m(torch.zeros(1, 8, cfg["input_dim"], device=DEV))
