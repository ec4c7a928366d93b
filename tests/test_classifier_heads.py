"""Utterance-level classifier heads (classifier 'global' / 'last', examples/speechcommand_v1/s0/conf/mdtc.yaml):
state-dict schema, the CPU oracle against the reference goldens, host packing and error behaviour without a GPU,
and on the GPU parity, cache identity with the linear head, determinism, launch count, kernel choice and the
PCM pipeline."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import kws_head_oracle as HO
from oracle import kws_oracle as O
from tests.conftest import golden, have_reference, reference_init_model
from tests.head_cases import (BATCH_B, BATCH_SEED, BATCH_T, FULL_SEED, FULL_T, HEAD_B, HEAD_CASES, HEAD_CHUNKS,
                              build_head_model, head_config)
from wekws_b200 import Mfcc, Pipeline, export_native, export_onnx, init_model, model_config, synth

CASES = list(HEAD_CASES)
TOL_POST = 1e-4


def _tol(ref):
    return TOL_POST * max(1.0, float(np.abs(ref).max()))


def _long_inputs(cfg, g):
    """The whole-utterance and batch inputs, regenerated from their seeds and checked against the stored sums."""
    idim = cfg["input_dim"]
    xf = synth.features(HEAD_B, FULL_T, idim, seed=FULL_SEED)
    xb = synth.features(BATCH_B, BATCH_T, idim, seed=BATCH_SEED)
    assert abs(float(xf.double().abs().sum()) - float(g["x_full_abs_sum"])) < 1e-9 * float(g["x_full_abs_sum"])
    assert abs(float(xb.double().abs().sum()) - float(g["x_batch_abs_sum"])) < 1e-9 * float(g["x_batch_abs_sum"])
    return xf, xb


# ----------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("case", CASES)
def test_state_dict_keys_shapes_and_weights_match_golden(case):
    g = golden("model_" + case)
    _, m = build_head_model(case, init_model)
    sd = m.state_dict()
    keys = sorted(sd)
    assert keys == [str(k) for k in g["keys"]]
    for k, shp in zip(keys, g["shapes"]):
        assert list(sd[k].shape) == [int(d) for d in shp[:sd[k].dim()]] and not shp[sd[k].dim():].any(), k
    assert abs(synth.state_digest(m) - float(g["digest"])) < 1e-6 * float(g["digest"])
    assert isinstance(m.activation, torch.nn.Identity) and m.head == HEAD_CASES[case][1]


def test_speech_command_mdtc_has_the_reference_key_count_and_loads_strict():
    cfg = head_config("mdtc_global")
    m = init_model(cfg)
    assert len(m.state_dict()) == 363
    g = golden("model_mdtc_global")
    other = {str(k): torch.randn(*[int(d) for d in s if d]) if any(s) else torch.tensor(0)
             for k, s in zip(g["keys"], g["shapes"])}
    m.load_state_dict(other, strict=True)
    if have_reference():
        _, ref = build_head_model("mdtc_global", reference_init_model())
        m.load_state_dict(ref.state_dict(), strict=True)
        assert synth.state_digest(m) == synth.state_digest(ref)


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference_golden(case):
    g = golden("model_" + case)
    cfg, m = build_head_model(case, init_model)
    sd = m.state_dict()
    cache = None
    for i in range(len(HEAD_CHUNKS)):
        y, cache = HO.kws_forward(sd, cfg, torch.from_numpy(g[f"x{i}"]), cache)
        assert np.abs(y.numpy() - g[f"y{i}"]).max() <= 1e-5 * max(1.0, float(np.abs(g[f"y{i}"]).max())), (case, i)
    n = len(HEAD_CHUNKS) - 1
    assert np.abs(cache.numpy() - g[f"c{n}"]).max() <= 1e-5 * max(1.0, float(np.abs(g[f"c{n}"]).max()))
    xf, xb = _long_inputs(cfg, g)
    yf, cf = HO.kws_forward(sd, cfg, xf, None)
    assert np.abs(yf.numpy() - g["y_full"]).max() <= 1e-5 * max(1.0, float(np.abs(g["y_full"]).max()))
    assert np.abs(cf.numpy() - g["c_full"]).max() <= 1e-5 * max(1.0, float(np.abs(g["c_full"]).max()))
    yb, _ = HO.kws_forward(sd, cfg, xb, None)
    assert np.abs(yb.numpy() - g["y_batch"]).max() <= 1e-5 * max(1.0, float(np.abs(g["y_batch"]).max()))


@pytest.mark.parametrize("case", CASES)
def test_pack_without_gpu_accepts_the_head_and_names_a_wrong_sized_tensor(case, native):
    _, m = build_head_model(case, init_model)
    h = m._build_handle(finalize=False)                 # create + set_head + every tensor + pack: no CUDA call
    assert h is not None
    m._release()
    lib = native.lib()
    cfg = m._native_config()
    h = C.c_void_p()
    native.check(lib.wekws_model_create(C.byref(cfg), C.byref(h)), "create")
    try:
        native.check(lib.wekws_model_set_head(h, native.HEAD_GLOBAL), "set_head")
        for name, t in m.state_dict().items():
            host = t.detach().float().contiguous()
            if name == "classifier.classifier.3.weight":
                host = host[:-1]                                             # one output row short
            native.check(lib.wekws_model_set_tensor(h, name.encode(), C.c_void_p(host.data_ptr()), host.numel()),
                         name)
        assert lib.wekws_model_pack(h) == -1
        assert "classifier.classifier.3.weight" in native.last_error()
        assert lib.wekws_model_set_head(h, 3) == -1
    finally:
        lib.wekws_model_destroy(h)


def test_heads_are_refused_behind_gru_and_fsmn_natively(native):
    lib = native.lib()
    for backbone in (native.BACKBONE_GRU, native.BACKBONE_FSMN):
        cfg = native.ModelConfig(backbone=backbone, idim=80, hdim=128, odim=11, num_layers=2)
        h = C.c_void_p()
        native.check(lib.wekws_model_create(C.byref(cfg), C.byref(h)), "create")
        try:
            assert lib.wekws_model_set_head(h, native.HEAD_LAST) == -1
            assert "last" in native.last_error()
            assert lib.wekws_model_set_head(h, native.HEAD_LINEAR) == 0
        finally:
            lib.wekws_model_destroy(h)


@pytest.mark.parametrize("head", ["global", "last"])
def test_init_model_errors_and_exporters(head, tmp_path):
    gru = model_config("gru", output_dim=11)
    gru["classifier"] = dict(type=head, dropout=0.5)
    with pytest.raises(NotImplementedError, match=head):
        init_model(gru)
    fsmn = model_config("fsmn", output_dim=11)
    fsmn["classifier"] = dict(type=head, dropout=0.1)
    with pytest.raises(NotImplementedError, match=head):
        init_model(fsmn)
    nodrop = model_config("mdtc", output_dim=11)
    nodrop["classifier"] = dict(type=head)
    with pytest.raises(KeyError):
        init_model(nodrop)
    one = model_config("mdtc", output_dim=1)               # no non-keyword class: a degenerate classifier
    one["classifier"] = dict(type=head, dropout=0.5)
    with pytest.raises(NotImplementedError, match="output_dim >= 2"):
        init_model(one)
    two = model_config("tcn", output_dim=2)
    two["classifier"] = dict(type=head, dropout=0.5)
    assert init_model(two).head == head
    cfg = model_config("mdtc", output_dim=11)
    cfg["classifier"] = dict(type=head, dropout=0.5)
    m = init_model(cfg).eval()
    with pytest.raises(NotImplementedError, match=head):
        export_native(m, str(tmp_path / "m.wkb"))
    with pytest.raises(NotImplementedError, match=head):
        export_onnx(m, str(tmp_path / "m.onnx"))
    with pytest.raises(IndexError):                        # softmax(2) of a 2-D output, as in the reference
        m.forward_softmax(torch.zeros(1, 5, 80))


# ----------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda:0"


@pytest.fixture(scope="module")
def head_models():
    cache = {}

    def get(case):
        if case not in cache:
            cfg, m = build_head_model(case, init_model)
            sd = {k: v.clone() for k, v in m.state_dict().items()}
            cache[case] = (cfg, m.to(DEV), sd)
        return cache[case]
    return get


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "fp32", "tensor"])
@pytest.mark.parametrize("case", CASES)
def test_gpu_matches_reference_golden(case, precision, head_models):
    g = golden("model_" + case)
    cfg, m, _ = head_models(case)
    m.precision = precision
    try:
        cache = torch.zeros(0, 0, 0)
        for i in range(len(HEAD_CHUNKS)):
            y, cache = m(torch.from_numpy(g[f"x{i}"]).to(DEV), cache)
            assert y.shape == (HEAD_B, cfg["output_dim"])
            assert np.abs(y.cpu().numpy() - g[f"y{i}"]).max() <= _tol(g[f"y{i}"]), (case, precision, i)
        n = len(HEAD_CHUNKS) - 1
        assert np.abs(cache.cpu().numpy() - g[f"c{n}"]).max() <= _tol(g[f"c{n}"])
        xf, xb = _long_inputs(cfg, g)
        yf, cf = m(xf.to(DEV))
        assert np.abs(yf.cpu().numpy() - g["y_full"]).max() <= _tol(g["y_full"]), (case, precision)
        assert np.abs(cf.cpu().numpy() - g["c_full"]).max() <= _tol(g["c_full"])
        yb, _ = m(xb.to(DEV))
        assert np.abs(yb.cpu().numpy() - g["y_batch"]).max() <= _tol(g["y_batch"]), (case, precision)
    finally:
        m.precision = "auto"


@pytest.mark.gpu
@pytest.mark.parametrize("B,T", [(1, 1), (5, 7), (3, 33), (7, 40), (2, 131), (64, 98)])
@pytest.mark.parametrize("case", CASES)
def test_gpu_matches_oracle_with_random_cache(case, B, T, head_models):
    cfg, m, sd = head_models(case)
    g = torch.Generator().manual_seed(1000 * B + T)
    x = torch.randn(B, T, cfg["input_dim"], generator=g)
    cache = 0.5 * torch.randn(B, m.hdim, m.backbone.padding, generator=g)
    y, c = m(x.to(DEV), cache.to(DEV))
    y_ref, c_ref = HO.kws_forward(sd, cfg, x, cache)
    assert y.shape == (B, cfg["output_dim"])
    assert (y.cpu() - y_ref).abs().max() <= _tol(y_ref.numpy()), (case, B, T)
    assert (c.cpu() - c_ref).abs().max() <= _tol(c_ref.numpy()), (case, B, T)


def _linear_twin(case, head_model):
    """A linear-head model with the head model's CMVN, preprocessing and backbone weights."""
    name, _, _, idim = HEAD_CASES[case]
    lin = init_model(model_config(name, input_dim=idim, output_dim=1)).eval()
    sd = head_model.state_dict()
    own = lin.state_dict()
    with torch.no_grad():
        for k, v in own.items():
            if not k.startswith("classifier."):
                v.copy_(sd[k].cpu())
    return lin.to(DEV)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["auto", "fp32"])
@pytest.mark.parametrize("case", CASES)
def test_gpu_cache_is_bitwise_that_of_the_linear_head(case, precision, head_models):
    cfg, m, _ = head_models(case)
    lin = _linear_twin(case, m)
    m.precision = lin.precision = precision
    try:
        g = torch.Generator().manual_seed(7)
        for B, T in ((3, 40), (2, 300), (BATCH_B, BATCH_T)):
            x = torch.randn(B, T, cfg["input_dim"], generator=g).to(DEV)
            cache = (0.5 * torch.randn(B, m.hdim, m.backbone.padding, generator=g)).to(DEV)
            _, c_head = m(x, cache)
            _, c_lin = lin(x, cache)
            # a TCN head runs the FP32 conv kernel; the linear TCN takes tcn_tc.cu under "auto"
            if HEAD_CASES[case][0] != "tcn" or precision == "fp32":
                assert torch.equal(c_head, c_lin), (case, precision, B, T)
    finally:
        m.precision = "auto"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_gpu_deterministic_launch_count_and_kernel_choice(case, head_models, native):
    cfg, m, _ = head_models(case)
    x = torch.randn(BATCH_B, BATCH_T, cfg["input_dim"], generator=torch.Generator().manual_seed(3)).to(DEV)
    y1, c1 = m(x)
    y2, c2 = m(x)
    torch.cuda.synchronize()
    assert torch.equal(y1, y2) and torch.equal(c1, c2)
    n0 = native.launch_count()
    m(x)
    torch.cuda.synchronize()
    if HEAD_CASES[case][0] == "mdtc":
        assert native.launch_count() - n0 == 2              # backbone kernel + head kernel
    assert m.uses_tensor_cores(98) == (case in ("mdtc_global", "mdtc_last"))
    with pytest.raises(ValueError):
        m(x[:, :0])
    with pytest.raises(IndexError):
        m.forward_softmax(x)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["mdtc_global", "mdtc_last", "tcn_global"])
def test_gpu_pipeline_mfcc_equals_model_on_mfcc_and_oracle(case, head_models):
    cfg, m, sd = head_models(case)
    pcm = synth.pcm_int16(3, 16000, seed=21)
    fe = Mfcc(80, 80)
    yp, cp = Pipeline(fe, m)(pcm.to(DEV))
    feats = fe(pcm.to(DEV))
    ym, cm = m(feats)
    assert yp.shape == (3, cfg["output_dim"])
    assert torch.equal(yp, ym) and torch.equal(cp, cm)
    ref_f = torch.stack([O.mfcc(pcm[b].float(), 80, 80) for b in range(3)])
    y_ref, _ = HO.kws_forward(sd, cfg, ref_f, None)
    assert (yp.cpu() - y_ref).abs().max() <= _tol(y_ref.numpy()), float((yp.cpu() - y_ref).abs().max())
    ys, _ = Pipeline(fe, m)(pcm.to(DEV), softmax=True)       # WEKWS_FWD_SOFTMAX: each row normalised
    assert (ys - ym.softmax(1)).abs().max() <= 1e-6
