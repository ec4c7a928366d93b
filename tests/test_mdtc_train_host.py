"""MDTC training without a device: the oracle against the reference's training-mode results
(tests/golden/mdtc_train.npz), the parameter order of the native entry points, their size and launch formulas, the
opt-in and every refusal that needs no device."""
import copy
import ctypes as C
import pickle
import re

import numpy as np
import pytest
import torch

from oracle import kws_mdtc_train_oracle as KM
from tests.cases import build_model
from wekws_b200 import _native, init_model, mdtc_train, model_config, synth

GOLDEN = np.load(__file__.rsplit("/", 1)[0] + "/golden/mdtc_train.npz")
NAMES = [str(n) for n in GOLDEN["names"]]
FLOOR = 2.0 ** -24
REFUSAL = ("wekws_b200.KWSModel is inference-only: call model.eval() first "
           "(training-mode BatchNorm/Dropout are not implemented)")


def golden_model(case):
    """(cfg, wekws_b200 model) of a golden case: the weights regenerated and checked against the fixture's digest."""
    cfg, model, _ = build_model(case, init_model)
    assert synth.state_digest(model) == float(GOLDEN[f"digest_{case}"])
    return cfg, model


def golden(name, key):
    return GOLDEN[f"{name}__{key}"]


def golden_feats(name, cfg):
    B, T, seed = (int(golden(name, k)) for k in ("B", "T", "seed"))
    x = synth.features(B, T, cfg["input_dim"], seed=seed, cmvn_like="cmvn" in cfg)
    assert x.double().sum().item() == float(golden(name, "feats_sum"))
    return x


def golden_up(name):
    """The float64 chain's upstream gradient, rounded to float32: what a float32 caller passes on."""
    return torch.from_numpy(golden(name, "up64")).float()


def golden_err32(name, n_params, n_running):
    """The reference's own float32-vs-float64 max error of each parameter gradient, running statistic, the logits."""
    e_g, e_r = golden(name, "err32_g"), golden(name, "err32_run")
    assert len(e_g) == n_params and len(e_r) == n_running
    return [float(e) for e in e_g], [float(e) for e in e_r], float(golden(name, "err32_l"))


def assert_within_rule(got, ref64, err32, what):
    """Each tensor: |value - float64| at most 8x the reference's own float32 error, plus 2^-24."""
    for i, (d, b, e) in enumerate(zip(got, ref64, err32)):
        d, b = d.detach().cpu().double(), b.detach().cpu().double()
        assert d.shape == b.shape, f"{what}: tensor {i}: shape {tuple(d.shape)} != {tuple(b.shape)}"
        err, bound = float((d - b).abs().max()), 8.0 * e + FLOOR
        assert err <= bound, f"{what}: tensor {i}: error {err:.3e} > bound {bound:.3e}"


def assert_digest(x64, stored, what, scale=0.0):
    """`stored` is the reference's float64 tensor as KM.digest: x64 must give the same fingerprint up to float64
    round-off (plus 2^-40 of `scale` per element: the round-off of the gradients that are zero in exact arithmetic,
    those of the biases a BatchNorm cancels)."""
    got, want = KM.digest(x64), torch.from_numpy(np.asarray(stored))
    tol = KM.digest_tolerance(x64, 2.0 ** -40 * scale)
    assert bool(((got - want).abs() <= tol).all()), f"{what}: digest {got.tolist()} != {want.tolist()}"


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    cfg, model = golden_model(str(golden(name, "case")))
    sd = model.state_dict()
    feats = golden_feats(name, cfg)
    bb = cfg["backbone"]
    names, rnames = KM.param_names(bb), KM.running_names(bb)
    e_g, e_r, e_l = golden_err32(name, len(names), len(rnames))
    # float64: the same upstream gradient as the reference's float64 chain
    y64, g64, r64, _ = KM.mdtc_train_grads(sd, cfg, feats, torch.from_numpy(golden(name, "up64")), torch.float64)
    torch.testing.assert_close(y64, torch.from_numpy(golden(name, "l64")), rtol=1e-12, atol=1e-14)
    scale = max(float(g.abs().max()) for g in g64)
    gd, rd = golden(name, "g64_digest"), golden(name, "run64_digest")
    assert len(gd) == len(g64) and len(rd) == len(rnames)
    for i, g in enumerate(g64):
        assert_digest(g, gd[i], f"{name}: gradient {i} ({names[i]})", scale)
    for j, k in enumerate(rnames):
        assert_digest(r64[k], rd[j], f"{name}: {k}")
    # float32: the logits, and everything under the rule the device is held to
    y32, g32, r32, _ = KM.mdtc_train_grads(sd, cfg, feats, golden_up(name), torch.float32)
    torch.testing.assert_close(y32, torch.from_numpy(golden(name, "logits")), rtol=1e-5, atol=1e-5)
    assert_within_rule(g32, g64, e_g, name)
    assert_within_rule([r32[k] for k in rnames], [r64[k] for k in rnames], e_r, name)
    assert_within_rule([y32], [y64], [e_l], name)


@pytest.mark.parametrize("case", ["mdtc", "mdtc_small", "mdtc_cmvn_logits"])
def test_param_order_is_named_parameters_order(case):
    cfg, model = golden_model(case)
    bb = cfg["backbone"]
    names = [n for n, _ in model.named_parameters()]
    assert mdtc_train.param_names(bb["num_stack"], bb["stack_size"]) == names == KM.param_names(bb)
    assert [n for n in model.state_dict() if n in dict(model.named_parameters())] == names
    assert len(mdtc_train.batch_norms(model)) == 3 * (1 + bb["num_stack"] * bb["stack_size"])


def config_handle(model):
    return _native.create("wekws_model_create", C.byref(model._native_config()))


@pytest.mark.parametrize("name", ["mdtc", "mdtc_small"])
def test_training_size_and_launch_formulas(name):
    model = init_model(model_config(name))
    bb = model.backbone
    L, Ch, K, idim, O = 1 + bb.num_stack * bb.stack_size, model.hdim, bb.kernel_size, model.idim, model.odim
    assert (L, Ch) == ((17, 64) if name == "mdtc" else (13, 32))
    h = config_handle(model)
    lib = _native.lib()
    try:
        assert lib.wekws_train_num_params(h) == 4 + 12 * L == len(list(model.parameters()))
        assert lib.wekws_train_forward_launches(h) == mdtc_train.forward_launches(L) == 2 + 3 * L
        assert lib.wekws_train_backward_launches(h) == mdtc_train.backward_launches(L) == 3 + 4 * L
        sliced = Ch * idim + Ch + L * (Ch * K + Ch + 2 * (Ch * Ch + Ch)) + O * Ch + O
        assert sliced == sum(p.numel() for n, p in model.named_parameters() if ".bn" not in n)
        for B, T in ((1, 2), (3, 5), (100, 200), (100, 1000)):
            M = B * T
            assert lib.wekws_train_saved_floats(h, B, T) == mdtc_train.saved_floats(L, Ch, B, T) \
                == 12 * L * Ch + M * Ch * (4 * L + 2)
            assert lib.wekws_train_workspace_bytes(h, B, T, 1) == 48 * 128 * Ch
            assert lib.wekws_train_workspace_bytes(h, B, T, 0) == 48 * 128 * Ch + 24 * M * Ch
            assert lib.wekws_train_backward_workspace_bytes(h, B, T) == 32 * 128 * Ch + 20 * M * Ch + 8 * 128 * sliced
    finally:
        lib.wekws_model_destroy(h)


def test_training_entry_point_refusals_without_a_device():
    lib = _native.lib()
    model = init_model(model_config("mdtc", activation="identity"))
    h = config_handle(model)
    try:
        assert lib.wekws_train_forward(h, None, None, 0, None, None, None, None, 0, None, 0, None, None, None, 1, None,
                                       1, 1, None) < 0
        assert "B * T >= 2" in _native.last_error()
        # MDTC has no Dropout: n_p must be 0
        p = (C.c_double * 1)(0.1)
        assert lib.wekws_train_forward(h, None, None, 0, None, None, None, None, 7, p, 1, None, None, None, 1, None,
                                       2, 3, None) < 0
        assert "n_p = 1, but the MDTC model has 0 Dropout probabilities" in _native.last_error()
        assert lib.wekws_train_backward(h, None, None, 0, None, None, None, None, None, 7, p, 1, 2, 3, None, None,
                                        None) < 0
        assert "n_p = 1, but the MDTC model has 0 Dropout probabilities" in _native.last_error()
        # its parameters travel with each call: the packed-handle entry points refuse it and name the right ones
        assert lib.wekws_model_load_params(h, None, 0, None) < 0 and "wekws_train_forward" in _native.last_error()
        assert lib.wekws_model_train_forward(h, None, None, None, None, 2, 3, None) < 0
        assert "wekws_train_forward" in _native.last_error()
        # the same entry points take the head model, with the head's numbers
        _native.invoke("wekws_model_set_head", h, _native.HEAD_GLOBAL)
        assert lib.wekws_train_num_params(h) == 6 + 12 * 17
        assert lib.wekws_train_backward_launches(h) == mdtc_train.head_backward_launches(17) == 4 + 4 * 17
    finally:
        lib.wekws_model_destroy(h)
    big = init_model(model_config("mdtc"))
    big.hdim = 128
    h = config_handle(big)
    try:
        assert lib.wekws_train_num_params(h) == 0 and "hidden_dim 128" in _native.last_error()
    finally:
        lib.wekws_model_destroy(h)


def head_config(head):
    cfg = model_config("mdtc", output_dim=3)
    cfg["classifier"] = dict(type=head, dropout=0.1)
    return cfg


def test_enable_training_per_config():
    for name, kw in (("mdtc", {}), ("mdtc_small", dict(input_dim=40)), ("mdtc", dict(activation="identity")),
                     ("mdtc", dict(output_dim=2))):
        model = init_model(model_config(name, **kw))
        assert model.enable_training() is model
    cfg, model = golden_model("mdtc_cmvn_logits")
    assert model.global_cmvn is not None and model.enable_training() is model
    model.global_cmvn.norm_var = False
    assert model.enable_training() is model
    fsmn = init_model(model_config("fsmn", activation="identity"))
    assert fsmn.enable_training() is fsmn and not fsmn._training_enabled          # no-op: FSMN needs no opt-in
    for name, match in (("tcn", "TCN backbone"), ("ds_tcn", "DS-TCN backbone"), ("gru", "GRU backbone")):
        with pytest.raises(NotImplementedError, match=match):
            init_model(model_config(name)).enable_training()
    for head in ("global", "last"):
        with pytest.raises(NotImplementedError, match=f"'{head}' head has Dropout"):
            init_model(head_config(head)).enable_training()
    with pytest.raises(NotImplementedError, match="output_dim <= 16"):
        init_model(model_config("mdtc", output_dim=17)).enable_training()


def test_opt_in_is_not_state_and_survives_copies():
    model = init_model(model_config("mdtc")).enable_training()
    assert not any("training" in k for k in model.state_dict())
    for other in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
        assert other._training_enabled
    fresh = init_model(model_config("mdtc"))
    fresh.load_state_dict(model.state_dict())
    assert not fresh._training_enabled


def test_refusals_without_a_device():
    model = init_model(model_config("mdtc")).train()
    x = torch.zeros(2, 4, 80)
    with pytest.raises(RuntimeError, match=re.escape(REFUSAL) + ".*enable_training"):
        model(x)                                               # no opt-in: the refusal, with a pointer
    model.enable_training()
    with pytest.raises(RuntimeError, match="forward_softmax has no training path"):
        model.forward_softmax(x)
    with torch.no_grad(), pytest.raises(RuntimeError, match="forward_softmax has no training path"):
        model.forward_softmax(x)
    with pytest.raises(ValueError, match="streaming cache"):
        model(x, torch.zeros(model.cache_shape(2)))
    with pytest.raises(ValueError, match="features that require grad"):
        model(x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match=re.escape("Expected more than 1 value per channel when training")):
        model(torch.zeros(1, 1, 80))
    ref = torch.nn.BatchNorm1d(64).train()                     # torch's own message for the same batch
    with pytest.raises(ValueError, match=re.escape("Expected more than 1 value per channel when training")):
        ref(torch.zeros(1, 64, 1))
    model.backbone.blocks[1].res_blocks[2].bn1.momentum = None
    with pytest.raises(ValueError, match="momentum=None"):
        model(x)
    model.backbone.blocks[1].res_blocks[2].bn1.momentum = 0.1
    with pytest.raises(RuntimeError, match="runs on CUDA"):   # past every refusal: only the device is missing
        model(x)
    model.eval()
    with pytest.raises(RuntimeError, match="runs on CUDA"):
        model(x, torch.zeros(model.cache_shape(2)))
