"""Speech-command MDTC training (the `global` / `last` head) without a device: the oracle and the Dropout mask against
the reference's training-mode results (tests/golden/mdtc_head_train.npz), the mask as its documented function, the
parameter order of the native entry points, their size and launch formulas, the opt-in and every refusal that needs no
device."""
import copy
import ctypes as C
import math
import pickle
import re

import numpy as np
import pytest
import torch

from oracle import kws_mdtc_head_train_oracle as KH
from oracle import kws_mdtc_train_oracle as KM
from tests.head_cases import build_head_model, head_config
from tests.test_mdtc_train_host import assert_digest, assert_within_rule
from wekws_b200 import _native, init_model, mdtc_train, model_config, synth
from wekws_b200.frontend import draw_seed

GOLDEN = np.load(__file__.rsplit("/", 1)[0] + "/golden/mdtc_head_train.npz")
NAMES = [str(n) for n in GOLDEN["names"]]


def golden(name, key):
    return GOLDEN[f"{name}__{key}"]


def golden_model(case):
    """(cfg, wekws_b200 model) of a golden case: the weights regenerated and checked against the fixture's digest."""
    cfg, model = build_head_model(case, init_model)
    assert synth.state_digest(model) == float(GOLDEN[f"digest_{case}"])
    return cfg, model


def golden_call(name):
    """(cfg, model with the call's p, features, mask, p) of a golden call; the mask regenerated from the seed a
    training forward draws after manual_seed(call_seed)."""
    cfg, model = golden_model(str(golden(name, "case")))
    p = float(golden(name, "p"))
    mtc = model.classifier.classifier[2]
    mtc.p = p
    B, T, seed = (int(golden(name, k)) for k in ("B", "T", "seed"))
    x = synth.features(B, T, cfg["input_dim"], seed=seed)
    assert x.double().sum().item() == float(golden(name, "feats_sum"))
    torch.manual_seed(int(golden(name, "call_seed")))
    dseed, p_drawn = mdtc_train.draw_head_dropout(model)
    assert p_drawn == p and dseed == int(golden(name, "dseed"))
    return cfg, model, x, KH.head_mask(dseed, B, p), p


@pytest.mark.parametrize("name", NAMES)
def test_oracle_and_mask_match_reference(name):
    cfg, model, feats, mask, p = golden_call(name)
    assert np.array_equal(np.packbits(mask), golden(name, "mask"))      # the mask the reference ran with
    sd = model.state_dict()
    bb = cfg["backbone"]
    names, rnames = KH.param_names(bb), KM.running_names(bb)
    e_g, e_r = [float(e) for e in golden(name, "err32_g")], [float(e) for e in golden(name, "err32_run")]
    assert len(e_g) == len(names) and len(e_r) == len(rnames)
    up64 = torch.from_numpy(golden(name, "up64"))
    y64, g64, r64, _ = KH.mdtc_head_train_grads(sd, cfg, feats, up64, mask, p, torch.float64)
    torch.testing.assert_close(y64, torch.from_numpy(golden(name, "l64")), rtol=1e-12, atol=1e-14)
    scale = max(float(g.abs().max()) for g in g64)
    gd, rd = golden(name, "g64_digest"), golden(name, "run64_digest")
    for i, g in enumerate(g64):
        assert_digest(g, gd[i], f"{name}: gradient {i} ({names[i]})", scale)
    for j, k in enumerate(rnames):
        assert_digest(r64[k], rd[j], f"{name}: {k}")
    y32, g32, r32, _ = KH.mdtc_head_train_grads(sd, cfg, feats, up64.float(), mask, p, torch.float32)
    torch.testing.assert_close(y32, torch.from_numpy(golden(name, "logits")), rtol=1e-5, atol=1e-5)
    assert_within_rule(g32, g64, e_g, name)
    assert_within_rule([r32[k] for k in rnames], [r64[k] for k in rnames], e_r, name)
    assert_within_rule([y32], [y64], [float(golden(name, "err32_l"))], name)


def test_stack_sum_is_the_mdtc_oracle_before_its_classifier():
    """The oracle's backbone is kws_mdtc_train_oracle's: its stack sum through the MDTC oracle's own classifier gives the
    MDTC oracle's logits."""
    cfg, model = golden_model("mdtc_small_last")
    sd = {k: v.double() for k, v in model.state_dict().items()}
    x = synth.features(2, 9, 40, seed=5).double()
    run_a = {k: sd[k].clone() for k in KM.running_names(cfg["backbone"])}
    run_b = {k: sd[k].clone() for k in KM.running_names(cfg["backbone"])}
    s, cache = KH.stack_sum(sd, cfg, x, run_a)
    W, b = torch.randn(3, 32, dtype=torch.float64), torch.randn(3, dtype=torch.float64)
    y, cache2 = KM.mdtc_train_logits(dict(sd, **{"classifier.linear.weight": W, "classifier.linear.bias": b}),
                                     dict(cfg, activation=dict(type="identity")), x, run_b)
    torch.testing.assert_close(torch.nn.functional.linear(s, W, b), y, rtol=1e-13, atol=1e-13)
    assert torch.equal(cache, cache2) and all(torch.equal(run_a[k], run_b[k]) for k in run_a)


def test_numpy_mask_is_the_documented_function():
    # restated by hand from the Philox words: counter (j // 4, 0, b, 256), component j % 4
    from oracle.kws_tcn_train_oracle import dropout_mask
    from oracle.kws_train_oracle import philox4x32_10
    seed, B, p = 0x0123456789ABCDEF, 3, 0.5
    m = dropout_mask(seed, B, 1, 64, 255, p)[:, 0, :]
    assert np.array_equal(m, KH.head_mask(seed, B, p))
    theta = math.ceil(p * 2 ** 24)
    for b in range(B):
        for j in range(64):
            w = philox4x32_10(np.array([j // 4, 0, b, 256], dtype=np.uint32), (seed & 0xFFFFFFFF, seed >> 32))
            assert bool(m[b, j]) == (int(w[j % 4]) >> 8 >= theta)
    assert 0.4 < m.mean() < 0.6
    assert KH.head_mask(seed, B, 0.0).all() and not KH.head_mask(seed, B, 1.0).any()
    # a stream apart from the TCN blocks' (counter word 3 = 1 + layer, layers 0..7)
    assert not any(np.array_equal(m, dropout_mask(seed, B, 1, 64, l, p)[:, 0, :]) for l in range(8))


@pytest.mark.parametrize("case", ["mdtc_global", "mdtc_last", "mdtc_small_last"])
def test_param_order_is_named_parameters_order(case):
    cfg, model = golden_model(case)
    bb = cfg["backbone"]
    names = [n for n, _ in model.named_parameters()]
    assert mdtc_train.head_param_names(bb["num_stack"], bb["stack_size"]) == names == KH.param_names(bb)
    assert names[-4:] == ["classifier.classifier.0.weight", "classifier.classifier.0.bias",
                          "classifier.classifier.3.weight", "classifier.classifier.3.bias"]
    L = 1 + bb["num_stack"] * bb["stack_size"]
    assert len(names) == 6 + 12 * L
    assert mdtc_train.head_dropout(model) is model.classifier.classifier[2]


def head_handle(model):
    h = _native.create("wekws_model_create", C.byref(model._native_config()))
    if model.head is not None:
        _native.invoke("wekws_model_set_head", h, {"global": _native.HEAD_GLOBAL, "last": _native.HEAD_LAST}[model.head])
    return h


@pytest.mark.parametrize("case,odim", [("mdtc_global", 11), ("mdtc_last", 36), ("mdtc_small_last", 4096)])
def test_training_size_and_launch_formulas(case, odim):
    cfg = head_config(case)
    cfg["output_dim"] = odim
    model = init_model(cfg)
    bb = model.backbone
    L, Ch, K, idim = 1 + bb.num_stack * bb.stack_size, model.hdim, bb.kernel_size, model.idim
    h = head_handle(model)
    lib = _native.lib()
    try:
        assert lib.wekws_train_num_params(h) == 6 + 12 * L == len(list(model.parameters()))
        assert lib.wekws_train_forward_launches(h) == mdtc_train.head_forward_launches(L) == 3 + 3 * L
        assert lib.wekws_train_backward_launches(h) == mdtc_train.head_backward_launches(L) == 4 + 4 * L
        sliced = Ch * idim + Ch + L * (Ch * K + Ch + 2 * (Ch * Ch + Ch))       # no classifier among the slice sums
        for B, T in ((1, 2), (3, 5), (100, 98), (256, 98)):
            M = B * T
            assert lib.wekws_train_saved_floats(h, B, T) == mdtc_train.head_saved_floats(L, Ch, B, T) \
                == 12 * L * Ch + M * Ch * (4 * L + 2) + B * (Ch + 64)
            assert lib.wekws_train_workspace_bytes(h, B, T, 1) == 48 * 128 * Ch
            assert lib.wekws_train_workspace_bytes(h, B, T, 0) == 48 * 128 * Ch + 24 * M * Ch
            assert lib.wekws_train_backward_workspace_bytes(h, B, T) == \
                32 * 128 * Ch + 24 * M * Ch + 8 * 128 * sliced + 512 * B
    finally:
        lib.wekws_model_destroy(h)


def test_training_entry_point_refusals_without_a_device():
    lib = _native.lib()
    # the same entry points give a linear-classifier model its own numbers and a head model the head's
    h = head_handle(init_model(model_config("mdtc")))
    try:
        assert lib.wekws_train_num_params(h) == 4 + 12 * 17
        assert lib.wekws_train_backward_launches(h) == mdtc_train.backward_launches(17)
        assert lib.wekws_train_saved_floats(h, 2, 3) == mdtc_train.saved_floats(17, 64, 2, 3)
    finally:
        lib.wekws_model_destroy(h)
    model = init_model(head_config("mdtc_global"))
    h = head_handle(model)
    p = lambda *ps: (C.c_double * len(ps))(*ps)
    try:
        assert lib.wekws_train_num_params(h) == 6 + 12 * 17
        assert lib.wekws_train_backward_launches(h) == mdtc_train.head_backward_launches(17)
        assert lib.wekws_train_saved_floats(h, 2, 3) == mdtc_train.head_saved_floats(17, 64, 2, 3)
        assert lib.wekws_train_forward(h, None, None, 0, None, None, None, None, 1, p(0.5), 1, None, None, None, 1,
                                       None, 1, 1, None) < 0
        assert "B * T >= 2" in _native.last_error()
        assert lib.wekws_train_forward(h, None, None, 0, None, None, None, None, 1, p(1.5), 1, None, None, None, 1,
                                       None, 2, 3, None) < 0
        assert "outside [0, 1]" in _native.last_error()
        assert lib.wekws_train_backward(h, None, None, 0, None, None, None, None, None, 1, p(0.5), 1, 2, 3, None, None,
                                        None) < 0
        assert "expected 210 parameters" in _native.last_error()
        # the head has one Dropout: n_p must be 1
        for ps in ((), (0.5, 0.5)):
            assert lib.wekws_train_forward(h, None, None, 0, None, None, None, None, 1, p(*ps), len(ps), None, None,
                                           None, 1, None, 2, 3, None) < 0
            assert f"n_p = {len(ps)}, but the MDTC (global / last head) model has 1 Dropout" in _native.last_error()
    finally:
        lib.wekws_model_destroy(h)
    for name, cfg, what in (("tcn", model_config("tcn"), "TCN model trains with the per-frame linear classifier"),
                            ("odim", dict(head_config("mdtc_global"), output_dim=4097), "output_dim 4097"),
                            ("sigmoid", None, "Identity activation")):
        m = init_model(cfg) if cfg is not None else init_model(head_config("mdtc_global"))
        if name == "tcn":
            m.classifier.head = "global"          # a TCN handle with a head
        if name == "sigmoid":
            m.activation = torch.nn.Sigmoid()
        h = head_handle(m)
        try:
            assert lib.wekws_train_num_params(h) == 0 and what in _native.last_error(), name
        finally:
            lib.wekws_model_destroy(h)


def test_enable_training_opt_in():
    for case in ("mdtc_global", "mdtc_last", "mdtc_small_last"):
        cfg = head_config(case)
        with pytest.raises(NotImplementedError, match=f"the '{cfg['classifier']['type']}' head has Dropout.*"
                                                      r"device_dropout=True"):
            init_model(cfg).enable_training()
        model = init_model(cfg)
        assert model.enable_training(device_dropout=True) is model
        assert model._training_enabled and model._device_dropout
        assert not any("training" in k or "dropout" in k for k in model.state_dict())
        for other in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
            assert other._training_enabled and other._device_dropout
    # output_dim: the head's own limit, not the per-frame classifier's 16
    for odim in (12, 36, 4096):
        init_model(dict(head_config("mdtc_global"), output_dim=odim)).enable_training(device_dropout=True)
    with pytest.raises(NotImplementedError, match=re.escape("with the 'global' head supports") + ".*output_dim <= 4096"):
        init_model(dict(head_config("mdtc_global"), output_dim=4097)).enable_training(device_dropout=True)
    with pytest.raises(NotImplementedError, match="output_dim <= 16"):
        init_model(model_config("mdtc", output_dim=17)).enable_training(device_dropout=True)
    # the heads behind TCN / DS-TCN stay refused, with or without device_dropout
    for name in ("tcn", "ds_tcn"):
        cfg = model_config(name, output_dim=3)
        cfg["classifier"] = dict(type="last", dropout=0.1)
        with pytest.raises(NotImplementedError, match="'last' head has Dropout and trains behind the MDTC backbone only"):
            init_model(cfg).enable_training(device_dropout=True)
    model = init_model(head_config("mdtc_global"))
    model.activation = torch.nn.Sigmoid()
    with pytest.raises(NotImplementedError, match="Identity activation"):
        model.enable_training(device_dropout=True)


def test_refusals_without_a_device():
    model = init_model(head_config("mdtc_global")).train()
    x = torch.zeros(2, 4, 80)
    with pytest.raises(RuntimeError, match=re.escape("inference-only") + ".*device_dropout=True"):
        model(x)                                               # no opt-in: the refusal, with a pointer
    model.enable_training(device_dropout=True)
    with pytest.raises(IndexError):
        model.forward_softmax(x)
    with pytest.raises(ValueError, match="streaming cache"):
        model(x, torch.zeros(model.cache_shape(2)))
    with pytest.raises(ValueError, match="features that require grad"):
        model(x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match=re.escape("Expected more than 1 value per channel when training")):
        model(torch.zeros(1, 1, 80))
    model.backbone.blocks[2].res_blocks[0].bn2.momentum = None
    with pytest.raises(ValueError, match="momentum=None"):
        model(x)
    model.backbone.blocks[2].res_blocks[0].bn2.momentum = 0.1
    with pytest.raises(RuntimeError, match="runs on CUDA"):   # past every refusal: only the device is missing
        model(x)
    # the p = 0 draw takes nothing from the generator
    mdtc_train.head_dropout(model).p = 0.0
    torch.manual_seed(3)
    assert mdtc_train.draw_head_dropout(model) == (0, 0.0)
    after = draw_seed()
    torch.manual_seed(3)
    assert after == draw_seed()
