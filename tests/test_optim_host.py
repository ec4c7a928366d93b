"""The device optimiser's host side (wekws_b200/optim.py, csrc/optim.cu): refusals, torch.optim.Adam's arguments and
defaults, the per-tensor scalars against torch's own, the C symbols and the workspace / launch formulas.  No GPU."""
import inspect
import math

import pytest
import torch

from wekws_b200 import Adam, _native, clip_grad_norm_, init_model, model_config
from wekws_b200.optim import adam_scalars
from tests.head_cases import head_config

# the parameter sets of every shipped training model: name -> config
PARAM_SETS = {
    "mdtc": lambda: model_config("mdtc"),
    "mdtc_small": lambda: model_config("mdtc_small"),
    "mdtc_head": lambda: head_config("mdtc_global"),
    "tcn": lambda: model_config("tcn"),
    "ds_tcn": lambda: model_config("ds_tcn"),
    "ds_tcn_2599": lambda: model_config("ds_tcn", output_dim=2599, activation="identity"),
    "gru": lambda: model_config("gru"),
    "fsmn_2599": lambda: model_config("fsmn", input_dim=400, output_dim=2599, activation="identity"),
}
TENSORS = {"mdtc": 208, "mdtc_small": 160, "mdtc_head": 210, "tcn": 20, "ds_tcn": 36, "ds_tcn_2599": 36, "gru": 12,
           "fsmn_2599": 28}

CLIP_MAX_TENSORS, ADAM_MAX_TENSORS, CLIP_MAX_CTAS, CLIP_ELEMS_PER_CTA = 1024, 512, 264, 2048


def test_param_sets_are_the_shipped_models():
    for name, cfg in PARAM_SETS.items():
        assert len(list(init_model(cfg()).parameters())) == TENSORS[name], name


@pytest.mark.parametrize("kw,word", [(dict(amsgrad=True), "amsgrad"), (dict(maximize=True), "maximize"),
                                     (dict(capturable=True), "capturable"), (dict(differentiable=True), "differentiable"),
                                     (dict(fused=True), "fused"), (dict(decoupled_weight_decay=True),
                                                                   "decoupled_weight_decay"),
                                     (dict(lr=torch.tensor(1e-3)), "tensor lr"),
                                     (dict(betas=(torch.tensor(0.9), torch.tensor(0.999))), "tensor betas")])
def test_adam_refuses_flags(kw, word):
    with pytest.raises(NotImplementedError, match=word):
        Adam([torch.nn.Parameter(torch.zeros(3))], **kw)


@pytest.mark.parametrize("param,word", [
    (torch.zeros(3, dtype=torch.float64), "torch.float64"),
    (torch.zeros(3, dtype=torch.bfloat16), "torch.bfloat16"),
    (torch.zeros(3, dtype=torch.complex64), "complex"),
    (torch.sparse_coo_tensor(torch.tensor([[0]]), torch.tensor([1.0]), (3,)), "sparse"),
    (torch.zeros(3), "cpu"),
])
def test_adam_refuses_parameters(param, word):
    with pytest.raises(NotImplementedError, match=word):
        Adam([torch.nn.Parameter(param, requires_grad=param.dtype.is_floating_point or param.is_complex())])


def test_adam_value_checks_as_torch():
    p = [torch.nn.Parameter(torch.zeros(3))]
    for kw in (dict(lr=-1.0), dict(eps=-1.0), dict(betas=(1.0, 0.999)), dict(betas=(0.9, -0.1)),
               dict(weight_decay=-1.0)):
        with pytest.raises(ValueError) as theirs:
            torch.optim.Adam(p, **kw)
        with pytest.raises(ValueError, match=str(theirs.value).replace("(", r"\(").replace(")", r"\)")):
            Adam(p, **kw)


def test_adam_signature_and_defaults_are_torch():
    ours, theirs = inspect.signature(Adam.__init__), inspect.signature(torch.optim.Adam.__init__)
    assert list(ours.parameters) == list(theirs.parameters)
    assert [p.default for p in ours.parameters.values()] == [p.default for p in theirs.parameters.values()]
    assert [p.kind for p in ours.parameters.values()] == [p.kind for p in theirs.parameters.values()]


def test_clip_refusals_and_empty():
    p = torch.nn.Parameter(torch.zeros(3))
    p.grad = torch.ones(3)
    for nt in (1, 3.0, math.inf):
        with pytest.raises(NotImplementedError, match="norm_type"):
            clip_grad_norm_([p], 1.0, norm_type=nt)
    with pytest.raises(ValueError, match="NaN"):
        clip_grad_norm_([p], math.nan)
    with pytest.raises(NotImplementedError, match="cpu"):
        clip_grad_norm_([p], 1.0)
    q = torch.nn.Parameter(torch.zeros(3))
    for params in ([q], q, []):
        got, want = clip_grad_norm_(params, 1.0), torch.nn.utils.clip_grad_norm_(params, 1.0)
        assert got.device == want.device and got.dtype == want.dtype and float(got) == float(want) == 0.0


def torch_scalars(groups, steps, skip=lambda step, i: False):
    """(lr, beta1, beta2, step, step_size, bc2_sqrt) as torch.optim.Adam(foreach=True) hands them to its foreach
    kernels, one record per tensor and step, captured from _foreach_div_ / _foreach_addcdiv_ on CPU tensors."""
    seen, rec = [], []
    div, addcdiv = torch._foreach_div_, torch._foreach_addcdiv_

    def cap_div(tensors, other):
        if isinstance(other, list) and other and isinstance(other[0], float):
            seen.append(list(other))
        return div(tensors, other)

    def cap_addcdiv(params, a, b, scalars=None, *args, **kw):
        seen.append(list(scalars))
        return addcdiv(params, a, b, scalars, *args, **kw)

    params = [[torch.nn.Parameter(torch.zeros(1)) for _ in range(2)] for _ in groups]
    opt = torch.optim.Adam([dict(params=ps, **g) for ps, g in zip(params, groups)], foreach=True)
    torch._foreach_div_, torch._foreach_addcdiv_ = cap_div, cap_addcdiv
    try:
        for step in range(steps):
            for gi, ps in enumerate(params):
                for i, p in enumerate(ps):
                    p.grad = None if skip(step, i) else torch.ones(1)
            seen.clear()
            opt.step()
            for gi, (ps, g) in enumerate(zip(params, groups)):
                live = [p for p in ps if p.grad is not None]
                bc2, ss = seen[2 * gi], seen[2 * gi + 1]
                for k, p in enumerate(live):
                    rec.append((g["lr"], g["betas"][0], g["betas"][1], opt.state[p]["step"].item(), ss[k], bc2[k]))
    finally:
        torch._foreach_div_, torch._foreach_addcdiv_ = div, addcdiv
    return rec


def test_host_scalars_are_torch_bit_for_bit():
    groups = [dict(lr=1e-3, betas=(0.9, 0.999)), dict(lr=2e-4, betas=(0.9, 0.98)),    # the recipes' and a common one
              dict(lr=10.0, betas=(0.0, 0.0)), dict(lr=1e-12, betas=(0.999999, 0.9999999)),
              dict(lr=0.5, betas=(0.5, 0.5))]
    rec = torch_scalars(groups, 10_000, skip=lambda step, i: i == 1 and step % 3 == 0)   # steps fall behind
    assert len(rec) > 5 * 10_000
    for lr, b1, b2, step, ss, bc in rec:
        got = adam_scalars(lr, b1, b2, step)
        assert got[0].hex() == ss.hex() and got[1].hex() == bc.hex(), (lr, b1, b2, step, got, ss, bc)


def test_abi_version_and_optimiser_symbols():
    lib = _native.lib()
    assert lib.wekws_abi_version() == _native.ABI_VERSION == 19
    for name in ("wekws_grad_clip_workspace_bytes", "wekws_grad_clip_launches", "wekws_grad_clip",
                 "wekws_adam_step_launches", "wekws_adam_step"):
        assert name in _native.SIGNATURES and getattr(lib, name) is not None


def clip_workspace_bytes(n, total):
    if n == 0 or total == 0:
        return 0
    ctas = min(CLIP_MAX_CTAS, max(1, -(-total // CLIP_ELEMS_PER_CTA)))
    return 8 * ctas * -(-n // CLIP_MAX_TENSORS)


def test_workspace_and_launch_formulas():
    lib = _native.lib()
    sizes = [(0, 0), (1, 1), (1, 2048), (1, 2049), (208, 159745), (28, 756133), (36, 965159), (1024, 540_672),
             (1025, 5000), (3000, 10 ** 8)]
    for n, total in sizes:
        assert lib.wekws_grad_clip_workspace_bytes(n, total) == clip_workspace_bytes(n, total), (n, total)
    assert lib.wekws_grad_clip_workspace_bytes(-1, 5) < 0 and lib.wekws_grad_clip_workspace_bytes(3, -5) < 0
    for n in (0, 1, 12, 208, 512, 513, 1024, 1025, 2049):
        assert lib.wekws_grad_clip_launches(n) == 2 * -(-n // CLIP_MAX_TENSORS)
        assert lib.wekws_adam_step_launches(n) == -(-n // ADAM_MAX_TENSORS)
    for name, cfg in PARAM_SETS.items():
        n = TENSORS[name]
        assert lib.wekws_grad_clip_launches(n) == 2 and lib.wekws_adam_step_launches(n) == 1, name


def test_native_argument_checks():
    lib = _native.lib()
    assert lib.wekws_grad_clip(None, None, -1, 1.0, None, None, None) != 0
    assert "bad tensor count" in _native.last_error()
    assert lib.wekws_grad_clip(None, None, 0, 1.0, None, None, None) == 0
    assert lib.wekws_adam_step(None, None, None, None, None, None, None, 2, 0.9, 0.999, 1e-8, 0.0, None) != 0
    assert "null argument" in _native.last_error()
