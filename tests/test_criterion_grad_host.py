"""CPU tests of the training-criterion gradients: the oracle's gradient helpers (oracle/kws_criterion_grad_oracle.py)
against the reference's own loss.py under autograd (tests/golden/criterion_grad.npz), the closed form the device
kernels implement against finite differences, and the device entry point's dispatch on requires_grad."""
import importlib

import numpy as np
import pytest
import torch

from oracle import kws_criterion_grad_oracle as KG
from oracle import kws_criterion_oracle as K
from tests.conftest import golden

C = importlib.import_module("wekws_b200.criterion")      # the module; the package exports its criterion() by that name

G = golden("criterion_grad")
NAMES = [str(n) for n in G["names"]]


def grad_inputs(name):
    """(type, logits, target, lengths, target_lengths, min_duration, upstream) of a golden call."""
    g = lambda k: torch.from_numpy(G[f"{name}__{k}"]) if f"{name}__{k}" in G else None
    return (str(G[f"{name}__type"]), g("logits"), g("target"), g("lengths"), g("target_lengths"),
            int(G[f"{name}__min_duration"]), float(G[f"{name}__up"]))


def same_bits(a, b):
    """Equal float arrays, NaN where the other has NaN."""
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.parametrize("name", NAMES)
def test_oracle_gradient_equals_golden(name):
    """Bit for bit in float32 and in float64: the oracle runs the reference's ops in the reference's order."""
    ctype, x, t, l, tl, md, up = grad_inputs(name)
    for dtype, suffix in ((torch.float32, ""), (torch.float64, "64")):
        loss, grad = KG.criterion_grad(ctype, x, t, l, tl, md, up, dtype)
        assert grad.dtype == dtype and same_bits(grad.numpy(), G[f"{name}__grad{suffix}"])
        assert same_bits(np.asarray(loss.item(), G[f"{name}__loss{suffix}"].dtype), G[f"{name}__loss{suffix}"])


def test_golden_covers_every_corner():
    g = lambda n: G[f"{n}__grad"]
    # ties split evenly; a min_duration mask removes tied frames from the payout; clamp ends; upstream gradient
    assert np.allclose(g("mp_ties")[0, :, 0], [-1 / 12, -1 / 12, 0, -1 / 12])
    assert np.array_equal(g("mp_ties_dur2")[0, :, 0], [0, 0, 0, -0.25])
    assert np.allclose(g("mp_ties_up3"), np.float32(3) * g("mp_ties"), rtol=2.0 ** -22, atol=0)
    assert np.array_equal(g("mp_clamp")[0, :, 0], np.float32([-2.5e7, 0])) and not g("mp_clamp")[1].any()
    assert g("mp_ties")[1, 3].tolist() == [0, 0] and g("mp_ties")[2, 2:].sum() == 0          # padding gets nothing
    tg = np.concatenate([G[f"{n}__target"] for n in NAMES if G[f"{n}__type"] == "max_pooling"])
    assert (tg < 0).any() and (tg >= 2).any()
    assert np.isnan(G["mp_nan__logits"]).any() and np.isnan(G["mp_nan__loss"]) and not np.isnan(g("mp_nan")).any()
    # ce: ignored rows are zero; every row ignored -> NaN loss, zero gradient
    assert not g("ce0")[G["ce0__target"] == -100].any() and g("ce0")[G["ce0__target"] != -100].all()
    assert np.isnan(G["ce_all_ignored__loss"]) and not g("ce_all_ignored").any()
    # ctc: repeats, empty labels, an utterance of no frames, padding rows zero, NaN rows of the infeasible utterance
    assert (G["ctc0__target_lengths"] == 0).any() and (G["ctc0__lengths"] == 0).any()
    lens = G["ctc0__lengths"]
    pad = np.arange(g("ctc0").shape[1])[None, :] >= lens[:, None]
    assert not g("ctc0")[pad].any() and np.isfinite(g("ctc0")).all()
    nan_rows = np.isnan(g("ctc_infeasible")).all(2)
    assert np.array_equal(np.isnan(g("ctc_infeasible")).any(2), nan_rows)
    want = np.zeros_like(nan_rows)
    want[1, :4] = True                                   # utterance 1: its 4 frames of T = 12; utterance 3 has none
    assert np.array_equal(nan_rows, want) and np.isinf(G["ctc_infeasible__loss"])
    assert G["ctc_1d__target"].ndim == 1 and G["ctc_1d_ragged__target_lengths"].max() > 1
    assert G["ctc_v2599__logits"].shape[2] == 2599 and G["ctc_v2599__up"] != 1


def test_ctc_closed_form_against_finite_differences():
    """(softmax - occupancy) / B, the formula of ctc_grad_kernel, checked in float64 against central differences of
    the loss and against autograd, independently of torch's ctc_loss backward."""
    gen = torch.Generator().manual_seed(3)
    B, T, V = 3, 6, 5
    x = torch.randn(B, T, V, generator=gen, dtype=torch.float64)
    tgt = torch.tensor([[2, 2, 4], [1, 3, 1], [0, 0, 0]])
    tl = torch.tensor([3, 3, 0])
    lens = torch.tensor([6, 4, 3])
    grad, total = KG.ctc_grad_closed_form(x, tgt, lens, tl)
    valid = torch.arange(T)[None, :] < lens[:, None]
    assert torch.allclose(total[valid], torch.ones(int(valid.sum()), dtype=torch.float64), atol=1e-12)
    assert not grad[~valid].any()
    assert float(grad.sum(2).abs().max()) < 1e-12          # softmax and occupancy both sum to 1 per frame
    loss = lambda v: K.ctc_loss(v, tgt, lens, tl)[0]
    eps = 1e-6
    num = torch.zeros_like(x)
    for i in range(x.numel()):
        d = torch.zeros(x.numel(), dtype=torch.float64)
        d[i] = eps
        d = d.view_as(x)
        num.view(-1)[i] = (loss(x + d) - loss(x - d)) / (2 * eps)
    assert float((grad - num).abs().max()) < 1e-8
    _, auto = KG.criterion_grad("ctc", x, tgt, lens, tl, dtype=torch.float64)
    assert float((grad - auto).abs().max()) < 1e-12


def test_closed_form_equals_golden_float64():
    for name in ("ctc0", "ctc_v2599"):
        ctype, x, t, l, tl, md, up = grad_inputs(name)
        grad, _ = KG.ctc_grad_closed_form(x, t, l, tl)
        assert float((grad * up - torch.from_numpy(G[f"{name}__grad64"])).abs().max()) < 1e-12


class Recorder:
    """Stands in for the native library: records the entry points called, computes nothing."""

    def __init__(self):
        self.calls = []

    def call(self, name, *args, device):
        self.calls.append(name)

    def __getattr__(self, name):                         # the *_workspace_bytes queries
        return lambda *a: 256


@pytest.fixture
def recorder(monkeypatch):
    r = Recorder()
    monkeypatch.setattr(C._native, "call", r.call)
    monkeypatch.setattr(C._native, "lib", lambda: r)
    monkeypatch.setattr(C, "_logits", lambda x, dim: x)   # the CUDA-only check; the dispatch below it is device-blind
    return r


def test_dispatch_on_requires_grad(recorder):
    """The forward-only entry points serve every call that cannot be differentiated; the autograd Functions are
    entered only when the logits require grad and grad mode is on."""
    calls = {"max_pooling": lambda x: C.criterion("max_pooling", x, torch.tensor([0, -1]), torch.tensor([5, 5])),
             "ce": lambda x: C.criterion("ce", x[:, 0], torch.tensor([0, 1]), None),
             "ctc": lambda x: C.criterion("ctc", x, torch.tensor([[1], [1]]), torch.tensor([5, 5]), torch.tensor([1, 1]))}
    for name, fn in calls.items():
        x = torch.rand(2, 5, 2)
        del recorder.calls[:]
        fn(x)
        with torch.no_grad():
            fn(x.clone().requires_grad_(True))
        assert recorder.calls == [f"wekws_criterion_{name}"] * 2
        del recorder.calls[:]
        loss, _ = fn(x.clone().requires_grad_(True))
        assert recorder.calls == [f"wekws_criterion_{name}_train"] and loss.requires_grad
        loss.backward()
        assert recorder.calls[1:] == [f"wekws_criterion_{name}_backward"]


def test_upstream_gradient_must_be_a_float32_scalar():
    x = torch.zeros(2, 3)
    assert C._upstream(torch.tensor(2.0), x).item() == 2.0
    for bad in (torch.ones(2), torch.tensor(1.0, dtype=torch.float64), torch.tensor(1)):
        with pytest.raises(ValueError):
            C._upstream(bad, x)


def test_cpu_logits_are_still_refused():
    x = torch.rand(2, 5, 2, requires_grad=True)
    with pytest.raises(ValueError):
        C.criterion("max_pooling", x, torch.tensor([0, -1]), torch.tensor([5, 5]))
    with pytest.raises(ValueError):
        C.criterion("ctc", x, torch.tensor([[1], [1]]), torch.tensor([5, 5]), torch.tensor([1, 1]))
