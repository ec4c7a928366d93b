"""FSMN training without a device: the oracle's gradients against the reference's (tests/golden/fsmn_train.npz), the
parameter order of the native entry points, their size formulas and refusals, and the eval kernel's SASS."""
import ctypes as C
import hashlib
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import kws_fsmn_train_oracle as KF
from tests.cases import FSMN_CASES, fsmn_config
from wekws_b200 import _native, fsmn_train, init_model, model_config, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "fsmn_train.npz"))
NAMES = [str(n) for n in GOLDEN["names"]]
# sha256 of the instruction text of the eval kernel's SASS (nvcc 12.9, sm_90a) before the training flag existed
FSMN_KERNEL_SASS_SHA256 = "12fd1125c220c48cecac7acbc1afb2f0e00e3968180547aceaa2ab58118964dc"
FSMN_KERNEL_SASS_LEN = 9944
FLOOR = 2.0 ** -24


def golden_model(mk):
    """(cfg, state_dict) of golden model `mk`."""
    case = str(GOLDEN[f"m{mk}__case"])
    cfg = fsmn_config(case)
    cfg["cmvn"] = dict(norm_var=bool(GOLDEN[f"m{mk}__norm_var"]))
    pre = f"sd_{case}__"
    sd = {k[len(pre):]: torch.from_numpy(GOLDEN[k]) for k in GOLDEN.files if k.startswith(pre)}
    return cfg, sd


def golden_feats(name):
    """The call's features, regenerated from their seed and checked against the sum the fixture pins."""
    B, T, seed = (int(GOLDEN[f"{name}__{k}"]) for k in ("B", "T", "seed"))
    x = synth.features(B, T, 40, seed=seed, cmvn_like=True)
    assert x.double().sum().item() == float(GOLDEN[f"{name}__feats_sum"])
    return x


def golden_up(name):
    """The float64 chain's upstream gradient, rounded to float32: what a float32 caller passes on."""
    return torch.from_numpy(GOLDEN[f"{name}__up64"]).float()


def golden_grads(name, n):
    """(float64 gradients, the reference's own float32-vs-float64 max error of each)."""
    return ([torch.from_numpy(GOLDEN[f"{name}__g64_{i}"]) for i in range(n)],
            [float(GOLDEN[f"{name}__err32_{i}"]) for i in range(n)])


def assert_within_rule(grads, g64, err32, what):
    """Each parameter: |gradient - float64| at most 8x the reference's own float32 error, plus 2^-24."""
    for i, (d, b, e) in enumerate(zip(grads, g64, err32)):
        d, b = d.cpu().double(), b.double()
        assert d.shape == b.shape
        err, bound = float((d - b).abs().max()), 8.0 * e + FLOOR
        assert err <= bound, f"{what}: parameter {i}: error {err:.3e} > bound {bound:.3e}"


@pytest.mark.parametrize("name", NAMES)
def test_oracle_grads_match_reference(name):
    cfg, sd = golden_model(int(GOLDEN[f"{name}__model"]))
    feats = golden_feats(name)
    n = len(KF.param_names(cfg["backbone"]["num_layers"]))
    ref64, err32 = golden_grads(name, n)
    # float64: the same upstream gradient as the reference's float64 chain
    _, g64 = KF.fsmn_grads(sd, cfg, feats, torch.from_numpy(GOLDEN[f"{name}__up64"]), torch.float64)
    for i in range(n):
        assert g64[i].shape == ref64[i].shape
        torch.testing.assert_close(g64[i], ref64[i], rtol=1e-10, atol=1e-12)
    # float32: the logits, and the gradients under the rule the device is held to
    y32, g32 = KF.fsmn_grads(sd, cfg, feats, golden_up(name), torch.float32)
    torch.testing.assert_close(y32, torch.from_numpy(GOLDEN[f"{name}__logits"]), rtol=1e-5, atol=1e-5)
    assert_within_rule(g32, ref64, err32, name)


@pytest.mark.parametrize("case", list(FSMN_CASES))
def test_param_order_is_state_dict_order(case):
    model = init_model(fsmn_config(case))
    params = dict(model.named_parameters())
    in_sd = [k for k in model.state_dict() if k in params]
    L = model.backbone.fsmn_layers
    assert fsmn_train.param_names(L) == in_sd == list(params) == KF.param_names(L)
    assert [str(n) for n in GOLDEN[f"names_{case}"]] == in_sd    # the reference's own model has this order too


def native_model(cfg):
    model = init_model(cfg)
    return model, _native.create("wekws_model_create", C.byref(model._native_config()))


@pytest.mark.parametrize("case", list(FSMN_CASES) + ["shipped"])
def test_training_saved_floats_and_workspace_formulas(case):
    cfg = model_config("fsmn", input_dim=400, output_dim=2599) if case == "shipped" else fsmn_config(case)
    model, h = native_model(cfg)
    try:
        lib = _native.lib()
        bb = model.backbone
        L, P, D = bb.fsmn_layers, bb.proj_dim, bb.linear_dim
        per_frame = bb.input_affine_dim + D + L * (2 * P + D) + bb.output_affine_dim
        assert fsmn_train.saved_floats_per_frame(bb) == per_frame
        assert lib.wekws_train_num_params(h) == 8 + 5 * L == len(list(model.parameters()))
        assert lib.wekws_train_backward_launches(h) == 8 + 5 * L
        numel = sum(p.numel() for p in model.parameters())
        width = max(bb.input_affine_dim, D, P, bb.output_affine_dim)
        for B, T in ((1, 1), (13, 5), (256, 200)):
            assert lib.wekws_train_saved_floats(h, B, T) == B * T * per_frame
            assert lib.wekws_train_backward_workspace_bytes(h, B, T) == 4 * (32 * numel + 2 * B * T * width)
    finally:
        _native.lib().wekws_model_destroy(h)


def test_shipped_config_sizes():
    bb = init_model(model_config("fsmn", input_dim=400, output_dim=2599)).backbone
    assert (bb.input_dim, bb.input_affine_dim, bb.linear_dim, bb.proj_dim, bb.fsmn_layers, bb.lorder, bb.rorder,
            bb.output_dim) == (400, 140, 250, 128, 4, 10, 2, 2599)
    assert fsmn_train.saved_floats_per_frame(bb) == 140 + 250 + 4 * (2 * 128 + 250) + 140


def test_training_entry_point_refusals_without_a_device():
    lib = _native.lib()
    model, h = native_model(fsmn_config("fsmn"))
    try:
        ptrs = (C.c_void_p * 23)()
        rc = lib.wekws_model_load_params(h, ptrs, 23, None)           # not finalized
        assert rc == -3 and "finalize" in _native.last_error()
        # FSMN trains on its packed weights: the entry points that take the parameters with each call refuse it and
        # name the right ones
        assert lib.wekws_train_forward(h, None, None, 0, None, None, None, None, 0, None, 0, None, None, None, 1, None,
                                       2, 3, None) < 0
        assert "wekws_model_train_forward" in _native.last_error()
        assert lib.wekws_train_backward(h, None, None, 0, None, None, None, None, None, 0, None, 0, 2, 3, None, None,
                                        None) < 0
        assert "wekws_model_backward" in _native.last_error()
        assert lib.wekws_train_workspace_bytes(h, 2, 3, 1) < 0 and lib.wekws_train_forward_launches(h) == 0
    finally:
        lib.wekws_model_destroy(h)
    _, hm = native_model(model_config("mdtc"))
    try:
        assert lib.wekws_train_num_params(hm) == 4 + 12 * 17                 # the MDTC model's own count
        assert lib.wekws_model_load_params(hm, None, 0, None) < 0 and "wekws_train_forward" in _native.last_error()
        assert lib.wekws_model_backward(hm, None, None, None, None, 2, 3, None, 0, None, None) < 0
        assert "wekws_train_backward" in _native.last_error()
    finally:
        lib.wekws_model_destroy(hm)


def taps_config(left_order, right_order):
    cfg = fsmn_config("fsmn")
    cfg["backbone"].update(left_order=left_order, right_order=right_order)
    return cfg


def test_more_taps_than_the_backward_holds_are_refused_by_every_training_entry_point():
    """The backward's memory kernel keeps one register per tap (32).  A 33-tap model is refused by the parameter
    pack, the training forward and the backward alike, naming the taps, before they look at anything else; a 32-tap
    model passes that check (and stops at the next: this handle is not finalized)."""
    lib = _native.lib()
    for lo, ro in ((21, 12), (1, 32), (60, 20)):
        _, h = native_model(taps_config(lo, ro))
        try:
            n = lib.wekws_train_num_params(h)
            assert lib.wekws_model_load_params(h, (C.c_void_p * n)(), n, None) < 0
            assert f"at most 32 memory taps (left_order + right_order), this one has {lo} + {ro}" in _native.last_error()
            assert lib.wekws_model_train_forward(h, None, None, None, None, 2, 3, None) < 0
            assert "wekws_model_train_forward: the FSMN model trains with at most 32" in _native.last_error()
            assert lib.wekws_model_backward(h, None, None, None, None, 2, 3, None, n, None, None) < 0
            assert "wekws_model_backward: the FSMN model trains with at most 32" in _native.last_error()
        finally:
            lib.wekws_model_destroy(h)
    _, h = native_model(taps_config(20, 12))
    try:
        assert lib.wekws_model_load_params(h, (C.c_void_p * 23)(), 23, None) == -3
        assert "finalize" in _native.last_error()
    finally:
        lib.wekws_model_destroy(h)


@pytest.mark.parametrize("name", ["mdtc", "tcn", "ds_tcn", "gru"])
def test_other_backbones_keep_refusing_training(name):
    model = init_model(model_config(name)).train()
    with pytest.raises(RuntimeError, match=re.escape("wekws_b200.KWSModel is inference-only: call model.eval() first "
                                                     "(training-mode BatchNorm/Dropout are not implemented)")):
        model(torch.zeros(1, 4, model.idim))


def test_fsmn_softmax_has_no_training_path():
    model = init_model(fsmn_config("fsmn")).train()
    with pytest.raises(RuntimeError, match="forward_softmax has no training path"):
        model.forward_softmax(torch.zeros(1, 4, model.idim))


def sass_instructions(obj, kernel):
    text = subprocess.run(["cuobjdump", "-sass", obj], check=True, capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out[cur] = []
            continue
        m = re.search(r"/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if cur and m:
            out[cur].append(m.group(1))
    found = [v for k, v in out.items() if k.endswith(f"{len(kernel)}{kernel}ENS_8FsmnArgsE")]
    assert len(found) == 1, sorted(out)
    return found[0]


def test_eval_kernel_sass_unchanged():
    obj = os.path.join(ROOT, "wekws_b200", "csrc", "fsmn.o")
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if shutil.which("cuobjdump") is None or not os.path.exists(obj):
        pytest.skip("needs cuobjdump and the built wekws_b200/csrc/fsmn.o")
    version = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout
    if "release 12.9" not in version:
        pytest.skip("the recorded SASS is nvcc 12.9's")
    ins = sass_instructions(obj, "fsmn_kernel")
    assert len(ins) == FSMN_KERNEL_SASS_LEN
    assert hashlib.sha256("\n".join(ins).encode()).hexdigest() == FSMN_KERNEL_SASS_SHA256
    assert len(sass_instructions(obj, "fsmn_train_kernel")) > 0
