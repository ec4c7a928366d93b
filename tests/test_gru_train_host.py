"""GRU training without a device: the oracle against the reference's own training-mode GRU model
(tests/golden/gru_train.npz), the parameter order, the size and launch-count formulas of the native library, the
opt-in, the refusals and limits, and the eval kernel's SASS."""
import copy
import ctypes as C
import hashlib
import os
import pickle
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import kws_gru_train_oracle as KG
from tests.test_mdtc_train_host import assert_digest, assert_within_rule
from wekws_b200 import _native, gru_train, init_model, model_config, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "gru_train.npz"))
NAMES = [str(n) for n in GOLDEN["names"]]
# sha256 and length of the instruction text of each eval instantiation gru_kernel<S> (nvcc 12.9, sm_90a) before the
# storing instantiation existed
GRU_KERNEL_SASS = {
    1: (1248, "caec90165144f462a9b051c392edf2619e2517a9db246dbde10fc00423029b5f"),
    2: (1320, "9b219de1dd6126ee0c09d384a7ade9d6eda5c125a1c67ae30ccf0d84250977d2"),
    4: (1424, "c1c1b6ad00ce0c74294d841b44199dc9ef3c2c4051420805e7d05d0abe5f17c8"),
    8: (1632, "53e270f04cebae47c12e9e1d4c95547d6e4548d4f59e37cfae9d5ed375c2b765"),
}


def golden(name, key):
    return GOLDEN[f"{name}__{key}"]


def golden_model(case):
    """(cfg, wekws_b200 model) of a golden case: the weights regenerated and checked against the fixture's digest."""
    cfg, model = KG.golden_model(case, init_model)
    assert synth.state_digest(model) == float(GOLDEN[f"digest_{case}"])
    return cfg, model


def golden_feats(name, cfg):
    B, T, seed = (int(golden(name, k)) for k in ("B", "T", "seed"))
    x = synth.features(B, T, cfg["input_dim"], seed=seed, cmvn_like="cmvn" in cfg)
    assert x.double().sum().item() == float(golden(name, "feats_sum"))
    return x


@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_reference(name):
    cfg, model = golden_model(str(golden(name, "case")))
    sd = model.state_dict()
    feats = golden_feats(name, cfg)
    names = KG.param_names(cfg["backbone"]["num_layers"])
    e_g = [float(e) for e in golden(name, "err32_g")]
    assert len(e_g) == len(names)
    up64 = torch.from_numpy(golden(name, "up64"))
    y64, g64 = KG.gru_grads(sd, cfg, feats, up64, torch.float64)
    torch.testing.assert_close(y64, torch.from_numpy(golden(name, "l64")), rtol=1e-12, atol=1e-14)
    scale = max(float(g.abs().max()) for g in g64)
    for i, g in enumerate(g64):
        assert_digest(g, golden(name, "g64_digest")[i], f"{name}: gradient {i} ({names[i]})", scale)
    y32, g32 = KG.gru_grads(sd, cfg, feats, up64.float(), torch.float32)
    torch.testing.assert_close(y32, torch.from_numpy(golden(name, "logits")), rtol=1e-5, atol=1e-6)
    assert_within_rule(g32, g64, e_g, name)
    assert_within_rule([y32], [y64], [float(golden(name, "err32_l"))], name)


@pytest.mark.parametrize("layers", [1, 2, 4])
def test_param_order_is_named_parameters_order(layers):
    cfg = model_config("gru")
    cfg["backbone"]["num_layers"] = layers
    names = [n for n, _ in init_model(cfg).named_parameters()]
    assert gru_train.param_names(layers) == names == KG.param_names(layers)


def config_handle(model):
    return _native.create("wekws_model_create", C.byref(model._native_config()))


@pytest.mark.parametrize("layers,idim,odim", [(1, 80, 1), (2, 40, 2), (4, 128, 37)])
def test_training_size_and_launch_formulas(layers, idim, odim):
    cfg = model_config("gru", input_dim=idim, output_dim=odim)
    cfg["backbone"]["num_layers"] = layers
    model = init_model(cfg)
    H = 128
    P = sum(p.numel() for p in model.parameters())
    h = config_handle(model)
    lib = _native.lib()
    try:
        assert lib.wekws_train_num_params(h) == 4 + 4 * layers == len(list(model.parameters()))
        assert lib.wekws_train_backward_launches(h) == 5 + 4 * layers
        for B, T in ((0, 5), (1, 1), (3, 7), (256, 200)):
            M = B * T
            assert lib.wekws_train_saved_floats(h, B, T) == M * gru_train.saved_floats_per_frame(layers) \
                == (1 + 5 * layers) * M * H
            assert lib.wekws_train_backward_workspace_bytes(h, B, T) == 4 * (32 * P + M * (8 * H + odim))
        # GRU trains on its packed weights: the entry points that take the parameters with each call refuse it and
        # name the right ones
        assert lib.wekws_train_backward(h, None, None, 0, None, None, None, None, None, 0, None, 0, 2, 3, None, None,
                                        None) < 0
        assert "the GRU model trains on the packed weights" in _native.last_error()
        assert "wekws_model_backward" in _native.last_error()
        assert lib.wekws_train_forward_launches(h) == 0 and "wekws_model_train_forward" in _native.last_error()
    finally:
        lib.wekws_model_destroy(h)
    # an MDTC handle: the same queries give the MDTC model's own numbers
    h = config_handle(init_model(model_config("mdtc")))
    try:
        assert lib.wekws_train_num_params(h) == 4 + 12 * 17 and lib.wekws_train_backward_launches(h) == 3 + 4 * 17
    finally:
        lib.wekws_model_destroy(h)


def test_opt_in():
    model = init_model(model_config("gru"))
    with pytest.raises(NotImplementedError, match=re.escape("GRU backbone")) as e:
        model.enable_training()
    assert "opt in with model.enable_training(bptt=True)" in str(e.value)
    with pytest.raises(NotImplementedError, match="GRU backbone"):
        model.enable_training(device_dropout=True)
    assert not model._training_enabled
    model.train()
    with pytest.raises(RuntimeError, match=re.escape("wekws_b200.KWSModel is inference-only: call model.eval() first "
                                                     "(training-mode BatchNorm/Dropout are not implemented) -- or "
                                                     "call model.enable_training(bptt=True)")):
        model(torch.zeros(1, 4, model.idim))
    assert model.enable_training(bptt=True) is model and model._training_enabled and model._bptt
    for other in (copy.deepcopy(model), pickle.loads(pickle.dumps(model))):
        assert other._training_enabled and other._bptt
    # past the opt-in a training-mode call goes on to the device checks (with grad and without)
    for grad in (True, False):
        with torch.set_grad_enabled(grad), pytest.raises(RuntimeError, match="runs on CUDA"):
            model(torch.zeros(1, 4, model.idim))
    with pytest.raises(RuntimeError, match="forward_softmax has no training path"):
        model.forward_softmax(torch.zeros(1, 4, model.idim))


def test_bptt_changes_nothing_for_other_backbones():
    mdtc = init_model(model_config("mdtc")).enable_training(bptt=True)
    assert mdtc._training_enabled and not mdtc._device_dropout
    with pytest.raises(NotImplementedError, match="device_dropout=True"):
        init_model(model_config("tcn")).enable_training(bptt=True)
    from tests.cases import fsmn_config
    fsmn = init_model(fsmn_config("fsmn"))
    assert fsmn.enable_training(bptt=True) is fsmn and not fsmn._training_enabled


def test_limits():
    def gru(layers=2, idim=40, hidden=128, **kw):
        cfg = model_config("gru", input_dim=idim, **kw)
        cfg["backbone"]["num_layers"] = layers
        cfg["hidden_dim"] = hidden
        return init_model(cfg)

    for layers in (1, 4):
        gru(layers=layers).enable_training(bptt=True)
    for idim in (1, 128):
        gru(idim=idim).enable_training(bptt=True)
    gru(output_dim=4096, activation="identity").enable_training(bptt=True)
    for kw, match in ((dict(layers=5), "1..4 layers"), (dict(idim=129), "input_dim 1..128"),
                      (dict(hidden=64), "hidden_dim 128")):
        with pytest.raises(NotImplementedError, match=re.escape(match)):
            gru(**kw).enable_training(bptt=True)
    model = gru()
    model.backbone.dropout = 0.1
    with pytest.raises(NotImplementedError, match="inter-layer Dropout"):
        model.enable_training(bptt=True)
    model = gru()
    model.activation = torch.nn.Tanh()
    with pytest.raises(NotImplementedError, match="Sigmoid or Identity"):
        model.enable_training(bptt=True)


def sass_instructions(obj):
    """{S: instruction lines} of the eval instantiations gru_kernel<S> in `obj`."""
    text = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            k = re.search(r"10gru_kernelILi(\d+)E(Lb0E)?EEvNS_7GruArgsE$", m.group(1))
            cur = int(k.group(1)) if k else None
            if cur is not None:
                out[cur] = []
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if cur is not None and m:
            out[cur].append(m.group(1))
    return out


def test_eval_kernel_sass_unchanged():
    obj = os.path.join(ROOT, "wekws_b200", "csrc", "gru.o")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if shutil.which("cuobjdump") is None or not os.path.exists(obj):
        pytest.skip("needs cuobjdump and the built wekws_b200/csrc/gru.o")
    version = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    got = sass_instructions(obj)
    assert sorted(got) == sorted(GRU_KERNEL_SASS)
    for S, (n, digest) in GRU_KERNEL_SASS.items():
        assert len(got[S]) == n, S
        assert hashlib.sha256("\n".join(got[S]).encode()).hexdigest() == digest, S
