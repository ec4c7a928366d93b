"""FSMN training on the device: training-mode logits, parameter gradients against the reference's (golden) and the
float64 oracle's, Executor.train end to end, determinism, launch counts and refusals."""
import numpy as np
import pytest
import torch

from oracle import kws_criterion_grad_oracle as KG
from oracle import kws_criterion_oracle as K
from oracle import kws_fsmn_train_oracle as KF
from oracle import kws_head_oracle as HO
from tests.cases import fsmn_config
from tests.test_config_sweep import FSMN_SMALL, build_config, build_row, inputs
from tests.test_fsmn_train_host import (GOLDEN, NAMES, assert_within_rule, golden_feats, golden_grads, golden_model,
                                        golden_up)
from wekws_b200 import _native, criterion, init_model, model_config
from wekws_b200.kws_model import GlobalCMVN

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SHIPPED = model_config("fsmn", input_dim=400, output_dim=2599, activation="identity")


def device_model(cfg, sd):
    """A wekws_b200 FSMN model on the device with the weights (and CMVN buffers) of `sd`."""
    model = init_model({k: v for k, v in cfg.items() if k != "cmvn"})
    if "global_cmvn.mean" in sd:
        model.global_cmvn = GlobalCMVN(sd["global_cmvn.mean"].clone(), sd["global_cmvn.istd"].clone(),
                                       cfg["cmvn"]["norm_var"])
    model.load_state_dict(sd)
    return model.to(DEV)


def train_step(model, feats, up):
    """Training-mode forward and backward of (logits * up).sum(); returns (logits, out_cache, grads)."""
    model.train()
    model.zero_grad(set_to_none=True)
    y, cache = model(feats)
    (y * up).sum().backward()
    return y.detach(), cache, [p.grad.detach().clone() for p in model.parameters()]


@pytest.mark.parametrize("name", NAMES)
def test_golden_logits_and_gradients(name):
    cfg, sd = golden_model(int(GOLDEN[f"{name}__model"]))
    model = device_model(cfg, sd)
    feats = golden_feats(name).to(DEV)
    up = golden_up(name).to(DEV)
    y, cache, grads = train_step(model, feats, up)
    with torch.no_grad():
        y_eval, cache_eval = model.eval()(feats)
    assert torch.equal(y.view(torch.int32), y_eval.view(torch.int32))       # the eval logits, bit for bit
    assert torch.equal(cache.view(torch.int32), cache_eval.view(torch.int32))
    torch.testing.assert_close(y.cpu(), torch.from_numpy(GOLDEN[f"{name}__logits"]), rtol=1e-4, atol=1e-5)
    g64, err32 = golden_grads(name, len(grads))
    assert_within_rule(grads, g64, err32, name)


def shipped_model(seed=3):
    torch.manual_seed(seed)
    return init_model(SHIPPED)


def test_shipped_logits_bitwise():
    model = shipped_model().to(DEV)
    feats = torch.randn(32, 200, 400, generator=torch.Generator().manual_seed(1)).to(DEV)
    model.train()
    y, cache = model(feats)
    assert y.requires_grad and not cache.requires_grad
    with torch.no_grad():
        y_eval, cache_eval = model.eval()(feats)
    assert torch.equal(y.detach().view(torch.int32), y_eval.view(torch.int32))
    assert torch.equal(cache.view(torch.int32), cache_eval.view(torch.int32))


def test_shipped_gradients_against_oracle():
    model = shipped_model()
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    gen = torch.Generator().manual_seed(2)
    feats = torch.randn(16, 150, 400, generator=gen)
    up = torch.randn(16, 150, 2599, generator=gen) * 1e-3
    up[3, 100:] = 0.0                                                         # padding rows of a CTC upstream
    _, g32 = KF.fsmn_grads(sd, SHIPPED, feats, up, torch.float32)
    _, g64 = KF.fsmn_grads(sd, SHIPPED, feats, up, torch.float64)
    _, _, grads = train_step(model.to(DEV), feats.to(DEV), up.to(DEV))
    err32 = [float((a.double() - b).abs().max()) for a, b in zip(g32, g64)]
    assert_within_rule(grads, g64, err32, "shipped")


class OracleFsmn(torch.nn.Module):
    """The oracle's FSMN forward as a torch model with the same parameters, in the same order."""

    def __init__(self, cfg, sd):
        super().__init__()
        self.cfg, self.names = cfg, KF.param_names(cfg["backbone"]["num_layers"])
        self.params = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone()) for n in self.names])
        self.buf = {k: v.clone() for k, v in sd.items() if k not in self.names}

    def forward(self, feats):
        return KF.fsmn_logits(dict(self.buf, **dict(zip(self.names, self.params))), self.cfg, feats), None


def oracle_criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    return K.criterion(type, logits, target, lengths, target_lengths, min_duration, validation)


def test_executor_train_end_to_end():
    cfg, sd = golden_model(0)
    gpu = device_model(cfg, sd)
    cpu = OracleFsmn(cfg, sd)
    gen = torch.Generator().manual_seed(8)
    batches = []
    for k in range(5):
        lens = torch.randint(12, 31, (8,), generator=gen)
        lens[0] = 30
        tl = torch.randint(1, 4, (8,), generator=gen)
        if k == 2:
            lens[3], tl[3] = 2, 3                                             # infeasible: the step is skipped
        batches.append(dict(feats=torch.randn(8, 30, 40, generator=gen) * 3 + 15,
                            target=torch.randint(1, 7, (8, 3), generator=gen), feats_lengths=lens, target_lengths=tl))
    args = {"criterion": "ctc", "grad_clip": 5.0}
    for model, crit, device in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV)):
        KG.train(crit, model, torch.optim.SGD(model.parameters(), lr=0.0), batches[:1], torch.device(device), args)
    for n, p, q in zip(cpu.names, cpu.parameters(), gpu.parameters()):
        assert torch.allclose(q.grad.cpu(), p.grad, rtol=1e-4, atol=1e-6), n
    logs = [KG.train(crit, model, torch.optim.Adam(model.parameters(), lr=1e-3), batches, torch.device(device), args)
            for model, crit, device in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV))]
    assert [s for _, s in logs[0]] == [s for _, s in logs[1]] == [k != 2 for k in range(5)]
    for (a, _), (b, _) in zip(*logs):
        assert (np.isinf(a) and np.isinf(b)) or abs(a - b) <= 1e-3 * abs(a)
    # after training, eval repacks from the host (the version counters moved): eval == oracle on the trained weights
    with torch.no_grad():
        y, _ = gpu.eval()(batches[0]["feats"].to(DEV))
        y_ref = cpu(batches[0]["feats"])[0]
    torch.testing.assert_close(y.cpu(), y_ref, rtol=1e-4, atol=1e-4)


def test_backward_is_deterministic():
    model = shipped_model().to(DEV).train()
    gen = torch.Generator().manual_seed(4)
    feats = torch.randn(8, 100, 400, generator=gen).to(DEV)
    up = torch.randn(8, 100, 2599, generator=gen).to(DEV)
    y, _ = model(feats)
    loss = (y * up).sum()
    g1 = torch.autograd.grad(loss, list(model.parameters()), retain_graph=True)
    g2 = torch.autograd.grad(loss, list(model.parameters()))
    for a, b in zip(g1, g2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_launch_counts_and_no_grad_path():
    cfg, sd = golden_model(1)
    model = device_model(cfg, sd)
    L = cfg["backbone"]["num_layers"]
    for T in (5, 64, 150):
        feats = torch.randn(3, T, 40, device=DEV)
        with torch.no_grad():
            n0 = _native.launch_count()
            y_eval, _ = model.eval()(feats)
            torch.cuda.synchronize()
            eval_launches = _native.launch_count() - n0
            n0 = _native.launch_count()
            y_nograd, _ = model.train()(feats)                                 # training mode without grad: eval
            torch.cuda.synchronize()
            assert _native.launch_count() - n0 == eval_launches == -(-T // 64)
            assert torch.equal(y_nograd.view(torch.int32), y_eval.view(torch.int32)) and not y_nograd.requires_grad
        n0 = _native.launch_count()
        y, _ = model(feats)
        torch.cuda.synchronize()
        assert _native.launch_count() - n0 == 1 + eval_launches                # pack + the eval path's chunks
        n0 = _native.launch_count()
        y.sum().backward()
        torch.cuda.synchronize()
        assert _native.launch_count() - n0 == 8 + 5 * L


def test_refusals():
    cfg, sd = golden_model(0)
    model = device_model(cfg, sd).train()
    feats = torch.randn(2, 10, 40, device=DEV)
    _, cache = model(feats)
    with pytest.raises(ValueError, match="streaming cache"):
        model(feats, cache)
    with pytest.raises(ValueError, match="features that require grad"):
        model(feats.clone().requires_grad_(True))
    y, _ = model(feats)
    g = torch.autograd.grad(y.sum(), list(model.parameters()), create_graph=True)
    assert not any(t.requires_grad for t in g)           # once_differentiable: the gradients are constants,
    with pytest.raises(RuntimeError):                    # so differentiating them again is refused
        g[0].sum().backward()
    w = model.backbone.out_linear2.linear.weight
    model.backbone.out_linear2.linear.weight = torch.nn.Parameter(w.detach().t().contiguous().t())
    with pytest.raises(ValueError, match="contiguous float32"):
        model(feats)
    for name in ("mdtc", "tcn", "ds_tcn", "gru"):
        other = init_model(model_config(name)).to(DEV).train()
        with pytest.raises(RuntimeError, match="inference-only"):
            other(torch.randn(1, 8, 80, device=DEV))


def test_33_taps_are_refused_before_any_launch_and_still_run_in_eval():
    """An FSMN with 21 + 12 memory taps, one more than the backward's memory kernel holds: a training-mode forward with
    grad raises, naming the taps, before its parameter pack or forward launches; the eval forward runs it."""
    cfg, model = build_config("fsmn", dict(FSMN_SMALL, left_order=21, right_order=12), init_model)
    sd64 = {k: v.double() for k, v in model.state_dict().items()}
    model = model.to(DEV)
    x, cache = inputs(cfg, 5, 40, seed=33)
    y, c = model(x.to(DEV), cache.to(DEV))
    y_ref, c_ref = HO.kws_forward(sd64, cfg, x.double(), cache.double())
    assert float((y.cpu().double() - y_ref).abs().max()) <= 2e-5 * max(1.0, float(y_ref.abs().max()))
    assert float((c.cpu().double() - c_ref).abs().max()) <= 2e-5 * max(1.0, float(c_ref.abs().max()))
    torch.cuda.synchronize()
    n0 = _native.launch_count()
    with pytest.raises(RuntimeError, match=r"at most 32 memory taps \(left_order \+ right_order\), this one has 21 \+ 12"):
        model.train()(x.to(DEV))
    torch.cuda.synchronize()
    assert _native.launch_count() == n0


def test_32_taps_gradients_against_oracle():
    """The backward's memory kernel with every tap register in use (20 + 12 taps): one training step's gradients
    against the float64 oracle, under the rule the golden cases are held to."""
    cfg, model = build_row("fsmn_l20_r12", init_model)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    gen = torch.Generator().manual_seed(32)
    feats = torch.randn(8, 100, cfg["input_dim"], generator=gen)
    up = torch.randn(8, 100, cfg["output_dim"], generator=gen)
    _, g32 = KF.fsmn_grads(sd, cfg, feats, up, torch.float32)
    _, g64 = KF.fsmn_grads(sd, cfg, feats, up, torch.float64)
    _, _, grads = train_step(model.to(DEV), feats.to(DEV), up.to(DEV))
    err32 = [float((a.double() - b).abs().max()) for a, b in zip(g32, g64)]
    assert_within_rule(grads, g64, err32, "fsmn_l20_r12")
