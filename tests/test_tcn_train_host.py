"""TCN / DS-TCN training without a device: the oracle and the numpy Dropout masks against the reference's own
training-mode model with those masks hooked into its nn.Dropout (tests/golden/tcn_train.npz), parameter order, the
size and launch-count formulas of the native library, the opt-in, the refusals and limits, and the MDTC training
kernels' SASS after the batch-norm helpers moved to train_common.cuh."""
import copy
import ctypes as C
import math
import os
import pickle
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import kws_tcn_train_oracle as KT
from tests.test_mdtc_train_host import assert_digest, assert_within_rule
from wekws_b200 import _native, init_model, mdtc_train, model_config, synth, tcn_train
from wekws_b200.frontend import draw_seed

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "wekws_b200", "csrc")
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "tcn_train.npz"))
NAMES = [str(n) for n in GOLDEN["names"]]
CASES = [("tcn", {}), ("ds_tcn", {}), ("ds_tcn", dict(activation="identity", output_dim=2599, input_dim=40))]


def golden(name, key):
    return GOLDEN[f"{name}__{key}"]


def golden_model(case):
    """(cfg, wekws_b200 model) of a golden case: the weights regenerated and checked against the fixture's digest."""
    cfg, model = KT.golden_model(case, init_model)
    assert synth.state_digest(model) == float(GOLDEN[f"digest_{case}"])
    return cfg, model


def golden_feats(name, cfg):
    B, T, seed = (int(golden(name, k)) for k in ("B", "T", "seed"))
    x = synth.features(B, T, cfg["input_dim"], seed=seed, cmvn_like="cmvn" in cfg)
    assert x.double().sum().item() == float(golden(name, "feats_sum"))
    return x


def golden_masks(name, model):
    """The call's Dropout masks regenerated from its seed: the seed a forward draws after manual_seed(call_seed)."""
    B, T = int(golden(name, "B")), int(golden(name, "T"))
    torch.manual_seed(int(golden(name, "call_seed")))
    seed = draw_seed()
    assert seed == int(golden(name, "dseed"))
    ps = [d.p for d in tcn_train.dropouts(model)]
    return KT.dropout_masks(seed, B, T, model.hdim, ps), ps


@pytest.mark.parametrize("name", NAMES)
def test_oracle_and_masks_match_reference(name):
    cfg, model = golden_model(str(golden(name, "case")))
    sd = model.state_dict()
    feats = golden_feats(name, cfg)
    masks, ps = golden_masks(name, model)
    # the numpy masks are the ones the reference ran with (its nn.Dropout hooked)
    assert np.array_equal(np.packbits(np.stack(masks)), golden(name, "masks"))
    bb = cfg["backbone"]
    names, rnames = KT.param_names(bb), KT.running_names(bb)
    e_g, e_r = [float(e) for e in golden(name, "err32_g")], [float(e) for e in golden(name, "err32_run")]
    assert len(e_g) == len(names) and len(e_r) == len(rnames)
    up64 = torch.from_numpy(golden(name, "up64"))
    y64, g64, r64, _ = KT.tcn_train_grads(sd, cfg, feats, up64, masks, ps, torch.float64)
    torch.testing.assert_close(y64, torch.from_numpy(golden(name, "l64")), rtol=1e-12, atol=1e-14)
    scale = max(float(g.abs().max()) for g in g64)
    gd, rd = golden(name, "g64_digest"), golden(name, "run64_digest")
    for i, g in enumerate(g64):
        assert_digest(g, gd[i], f"{name}: gradient {i} ({names[i]})", scale)
    for j, k in enumerate(rnames):
        assert_digest(r64[k], rd[j], f"{name}: {k}")
    y32, g32, r32, _ = KT.tcn_train_grads(sd, cfg, feats, up64.float(), masks, ps, torch.float32)
    torch.testing.assert_close(y32, torch.from_numpy(golden(name, "logits")), rtol=1e-5, atol=1e-5)
    assert_within_rule(g32, g64, e_g, name)
    assert_within_rule([r32[k] for k in rnames], [r64[k] for k in rnames], e_r, name)
    assert_within_rule([y32], [y64], [float(golden(name, "err32_l"))], name)


def config_handle(model):
    return _native.create("wekws_model_create", C.byref(model._native_config()))


@pytest.mark.parametrize("name,kw", CASES)
def test_param_order_is_named_parameters_order(name, kw):
    model = init_model(model_config(name, **kw))
    bb = model_config(name, **kw)["backbone"]
    names = [n for n, _ in model.named_parameters()]
    assert tcn_train.param_names(bb["num_layers"], bb["ds"]) == names == KT.param_names(bb)
    assert len(tcn_train.batch_norms(model)) == (2 if bb["ds"] else 1) * bb["num_layers"]
    assert [f"backbone.network.{l}.cnn.{j}.{s}" for l in range(bb["num_layers"])
            for j in ((1, 4) if bb["ds"] else (1,)) for s in ("running_mean", "running_var")] == \
        KT.running_names(bb)
    assert all(isinstance(d, torch.nn.Dropout) for d in tcn_train.dropouts(model))


def wg_splits(N, Qp, M):
    tiles = -(-N // 64) * -(-Qp // 64)
    return max(1, min(-(-264 // tiles), max(1, M // 256), 64))


@pytest.mark.parametrize("name,kw", CASES)
def test_training_size_and_launch_formulas(name, kw):
    model = init_model(model_config(name, **kw))
    bb = model.backbone
    L, Ch, K, idim, O, ds = bb.num_layers, model.hdim, bb.kernel_size, model.idim, model.odim, bb.ds
    h = config_handle(model)
    lib = _native.lib()
    try:
        assert lib.wekws_train_num_params(h) == 4 + (8 if ds else 4) * L == len(list(model.parameters()))
        assert lib.wekws_train_forward_launches(h) == tcn_train.forward_launches(L, ds) == 2 + (2 if ds else 1) * L
        assert lib.wekws_train_backward_launches(h) == tcn_train.backward_launches(L, ds) == 4 + (3 if ds else 2) * L
        for B, T in ((1, 2), (3, 5), (256, 200)):
            M = B * T
            nbn = (2 if ds else 1) * L
            assert lib.wekws_train_saved_floats(h, B, T) == tcn_train.saved_floats(L, Ch, ds, B, T) \
                == 4 * nbn * Ch + M * Ch * (1 + L * (3 if ds else 2))
            assert lib.wekws_train_workspace_bytes(h, B, T, 1) == 32 * 128 * Ch
            assert lib.wekws_train_workspace_bytes(h, B, T, 0) == 32 * 128 * Ch + 16 * M * Ch
            jobs = [(Ch, idim + 1), (O, Ch + 1)] + [(Ch, Ch + 1) if ds else (Ch, K * Ch + 1)] * L
            part = sum(wg_splits(n, q, M) * n * q for n, q in jobs) + (128 * Ch * (K + 1) * L if ds else 0)
            assert lib.wekws_train_backward_workspace_bytes(h, B, T) == 32 * 128 * Ch + 16 * M * Ch + 8 * part
    finally:
        lib.wekws_model_destroy(h)


def test_numpy_mask_is_the_documented_function():
    # one element restated by hand from the Philox words: counter (c // 4, t, b, 1 + layer), component c % 4
    from oracle.kws_train_oracle import philox4x32_10
    seed, B, T, C_, layer, p = 0xDEADBEEF12345678, 2, 3, 64, 2, 0.3
    m = KT.dropout_mask(seed, B, T, C_, layer, p)
    theta = math.ceil(p * 2 ** 24)
    for b, t, c in ((0, 0, 0), (1, 2, 63), (1, 1, 6)):
        w = philox4x32_10(np.array([c // 4, t, b, 1 + layer], dtype=np.uint32), (seed & 0xFFFFFFFF, seed >> 32))
        assert bool(m[b, t, c]) == (int(w[c % 4]) >> 8 >= theta)
    assert KT.dropout_mask(seed, B, T, C_, layer, 0.0).all() and not KT.dropout_mask(seed, B, T, C_, layer, 1.0).any()
    assert not np.array_equal(m, KT.dropout_mask(seed, B, T, C_, layer + 1, p))
    assert float(KT.scale(0.1, torch.float32)) == float(np.float32(1.0) / np.float32(0.9))


def test_opt_in():
    for name in ("tcn", "ds_tcn"):
        label = "DS-TCN" if name == "ds_tcn" else "TCN"
        with pytest.raises(NotImplementedError, match=f"{label} backbone.*device_dropout=True"):
            init_model(model_config(name)).enable_training()
        model = init_model(model_config(name))
        assert model.enable_training(device_dropout=True) is model and model._training_enabled
        assert not any("training" in k or "dropout" in k for k in model.state_dict())
        for other in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
            assert other._training_enabled and other._device_dropout
    for name in ("mdtc", "fsmn"):                                       # accepted, no effect
        kw = dict(activation="identity") if name == "fsmn" else {}
        model = init_model(model_config(name, **kw))
        assert model.enable_training(device_dropout=True) is model
    with pytest.raises(NotImplementedError, match="GRU backbone"):
        init_model(model_config("gru")).enable_training(device_dropout=True)
    cfg = model_config("ds_tcn", output_dim=3)
    cfg["classifier"] = dict(type="global", dropout=0.1)
    with pytest.raises(NotImplementedError, match="'global' head has Dropout"):
        init_model(cfg).enable_training(device_dropout=True)


def test_training_limits_and_refusals_without_a_device():
    for kw, what in ((dict(output_dim=4097), "output_dim <= 4096"), (dict(input_dim=129), "input_dim <= 128")):
        with pytest.raises(NotImplementedError, match=re.escape(what)):
            init_model(model_config("ds_tcn", **kw)).enable_training(device_dropout=True)
    cfg = model_config("tcn")
    cfg["backbone"]["num_layers"] = 9
    with pytest.raises(NotImplementedError, match="1..8 layers"):
        init_model(cfg).enable_training(device_dropout=True)
    lib = _native.lib()
    h = config_handle(init_model(model_config("tcn", output_dim=4097)))
    try:
        assert lib.wekws_train_num_params(h) == 0 and "output_dim <= 4096" in _native.last_error()
    finally:
        lib.wekws_model_destroy(h)
    tcn = init_model(model_config("tcn"))
    L = tcn.backbone.num_layers
    h = config_handle(tcn)
    try:
        assert lib.wekws_train_backward_launches(h) == tcn_train.backward_launches(L, False)
        # one Dropout probability per block: n_p must be L
        for n_p in (0, L - 1, L + 1):
            ps = (C.c_double * n_p)(*[0.1] * n_p)
            assert lib.wekws_train_forward(h, None, None, 0, None, None, None, None, 1, ps, n_p, None, None, None, 1,
                                           None, 2, 3, None) < 0
            assert f"n_p = {n_p}, but the TCN / DS-TCN model has {L} Dropout" in _native.last_error()
            assert lib.wekws_train_backward(h, None, None, 0, None, None, None, None, None, 1, ps, n_p, 2, 3, None,
                                            None, None) < 0
            assert f"n_p = {n_p}, but the TCN / DS-TCN model has {L} Dropout" in _native.last_error()
    finally:
        lib.wekws_model_destroy(h)
    h = config_handle(init_model(model_config("mdtc")))
    try:
        assert lib.wekws_train_backward_launches(h) == mdtc_train.backward_launches(17)
    finally:
        lib.wekws_model_destroy(h)
    model = init_model(model_config("ds_tcn")).enable_training(device_dropout=True).train()
    x = torch.zeros(2, 4, 80)
    with pytest.raises(RuntimeError, match="forward_softmax has no training path"):
        model.forward_softmax(x)
    with pytest.raises(ValueError, match="streaming cache"):
        model(x, torch.zeros(model.cache_shape(2)))
    with pytest.raises(ValueError, match="features that require grad"):
        model(x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match=re.escape("Expected more than 1 value per channel when training")):
        model(torch.zeros(1, 1, 80))
    model.backbone.network[2].cnn[4].momentum = None
    with pytest.raises(ValueError, match="momentum=None"):
        model(x)
    model.backbone.network[2].cnn[4].momentum = 0.1
    with pytest.raises(RuntimeError, match="runs on CUDA"):
        model(x)
    bare = init_model(model_config("tcn")).train()
    with pytest.raises(RuntimeError, match=re.escape("inference-only") + ".*device_dropout=True"):
        bare(x)


@pytest.mark.skipif(shutil.which("cuobjdump") is None and not os.path.exists("/usr/local/cuda/bin/cuobjdump"),
                    reason="needs cuobjdump")
def test_mdtc_training_sass_is_unchanged_by_the_shared_header(tmp_path):
    """mdtc_train.cu includes train_common.cuh for the batch-statistics helpers it used to define itself; its kernels
    compile to the instructions whose digest tests/golden/mdtc_train_sass.sha256 holds (the SASS before the move)."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    obj = tmp_path / "mdtc_train.o"
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler",
                    "-fPIC", "--expt-relaxed-constexpr", "-c", os.path.join(CSRC, "mdtc_train.cu"), "-o", str(obj)],
                   check=True, capture_output=True)
    sass = subprocess.run([cuobjdump, "-sass", str(obj)], check=True, capture_output=True, text=True).stdout
    got = [re.sub(r"_GLOBAL__N__[0-9a-f]+_[0-9]+_[a-z_]+_cu_[0-9a-f]+", "ANON", l) for l in sass.splitlines()
           if l.strip() and re.search(r"/\*[0-9a-f]{4}\*/", l)]
    import hashlib
    digest = hashlib.sha256("\n".join(got).encode()).hexdigest()
    with open(os.path.join(ROOT, "tests", "golden", "mdtc_train_sass.sha256")) as f:
        assert digest == f.read().split()[0]
