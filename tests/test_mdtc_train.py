"""MDTC training on the device: logits, running statistics and parameter gradients against float64 (the oracle,
pinned to the reference by tests/test_mdtc_train_host.py), Executor.train end to end, determinism, the no_grad path,
eval after a step, launch counts, edge shapes and refusals."""
import copy

import pytest
import torch

from oracle import kws_criterion_grad_oracle as KG
from oracle import kws_criterion_oracle as K
from oracle import kws_mdtc_train_oracle as KM
from tests.test_mdtc_train_host import (NAMES, assert_within_rule, golden, golden_err32, golden_feats, golden_model,
                                        golden_up)
from wekws_b200 import _native, criterion, init_model, mdtc_train, model_config, synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def running(model):
    return [t for bn in mdtc_train.batch_norms(model) for t in (bn.running_mean, bn.running_var)]


def train_step(model, feats, up):
    """Training-mode forward and backward of (logits * up).sum(): (logits, out_cache, grads)."""
    model.enable_training().train()
    model.zero_grad(set_to_none=True)
    y, cache = model(feats)
    (y * up).sum().backward()
    return y.detach(), cache, [p.grad.detach().clone() for p in model.parameters()]


def check_against_oracle(model, sd, cfg, feats, up, what, floor=0.0):
    """One device step against the float64 oracle, under the rule with the float32 oracle's own error on the same
    device as the unit: torch with its default settings, whose cuDNN convolutions may take TF32 (plus `floor` times
    the tensor's largest float64 magnitude).  The golden cases hold the kernels to the reference's CPU float32 error."""
    bb = cfg["backbone"]
    y64, g64, r64, c64 = KM.mdtc_train_grads(sd, cfg, feats, up, torch.float64, device=DEV)
    y32, g32, r32, c32 = KM.mdtc_train_grads(sd, cfg, feats, up, torch.float32, device=DEV)
    rn = KM.running_names(bb)
    y, cache, grads = train_step(model, feats.to(DEV), up.to(DEV))
    err = lambda a, b: float((a.double() - b).abs().max()) + floor / 8 * float(b.abs().max())
    assert_within_rule(grads, g64, [err(a, b) for a, b in zip(g32, g64)], what + " gradients")
    assert_within_rule(running(model), [r64[k] for k in rn], [err(r32[k], r64[k]) for k in rn], what + " running")
    assert_within_rule([y], [y64], [err(y32, y64)], what + " logits")
    assert_within_rule([cache], [c64], [err(c32, c64)], what + " out_cache")


@pytest.mark.parametrize("name", NAMES)
def test_golden_cases(name):
    cfg, model = golden_model(str(golden(name, "case")))
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    bb = cfg["backbone"]
    model = model.to(DEV).enable_training()
    feats = golden_feats(name, cfg)
    counts = [int(bn.num_batches_tracked) for bn in mdtc_train.batch_norms(model)]
    y, _, grads = train_step(model, feats.to(DEV), golden_up(name).to(DEV))
    assert [int(bn.num_batches_tracked) for bn in mdtc_train.batch_norms(model)] == [c + 1 for c in counts]
    # the float64 values: the oracle's, on the reference's own upstream gradient (the fixture pins them to float32)
    y64, g64, r64, _ = KM.mdtc_train_grads(sd, cfg, feats, torch.from_numpy(golden(name, "up64")), torch.float64)
    e_g, e_r, e_l = golden_err32(name, len(grads), len(KM.running_names(bb)))
    assert_within_rule(grads, g64, e_g, name)
    assert_within_rule(running(model), [r64[k] for k in KM.running_names(bb)], e_r, name)
    assert_within_rule([y], [y64], [e_l], name)


def shipped_model(name, seed=3):
    cfg = model_config(name)
    model = synth.randomize_(init_model(cfg), seed=seed)
    return cfg, model, {k: v.clone() for k, v in model.state_dict().items()}


@pytest.mark.parametrize("name", ["mdtc", "mdtc_small"])
def test_shipped_sizes_against_oracle(name):
    cfg, model, sd = shipped_model(name)
    gen = torch.Generator().manual_seed(5)
    B, T = 100, 200
    feats = torch.randn(B, T, 80, generator=gen)
    lens = torch.randint(100, T + 1, (B,), generator=gen)
    up = torch.randn(B, T, 1, generator=gen) * 1e-2
    up[torch.arange(T)[None, :] >= lens[:, None]] = 0.0                      # padding rows of a pooled loss
    check_against_oracle(model.to(DEV), sd, cfg, feats, up, f"{name} B={B} T={T}")


@pytest.mark.parametrize("B,T", [(1, 37), (3, 1), (5, 7), (2, 97)])
def test_edge_shapes(B, T):
    """One utterance; one frame per utterance (3 rows of batch statistics); fewer frames than the kernel taps; a length
    that is no multiple of any row tile.  The rule gets a floor of 2^-20 of each tensor's largest magnitude: with a few
    hundred rows at most, one tensor's float32 error can be far below its usual size (the classifier bias gradient of the
    97-frame case: 3.9e-8 for torch's float32, 9.1e-7 here)."""
    cfg, model, sd = shipped_model("mdtc_small", seed=9)
    gen = torch.Generator().manual_seed(B * 1000 + T)
    feats = torch.randn(B, T, 80, generator=gen)
    up = torch.randn(B, T, 1, generator=gen)
    check_against_oracle(model.to(DEV), sd, cfg, feats, up, f"B={B} T={T}", floor=2.0 ** -20)


class OracleMdtc(torch.nn.Module):
    """The oracle's training forward as a torch model with the same parameters, in the same order."""

    def __init__(self, cfg, sd):
        super().__init__()
        self.cfg, self.names = cfg, KM.param_names(cfg["backbone"])
        self.params = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone()) for n in self.names])
        self.buf = {k: v.clone() for k, v in sd.items() if k not in self.names}

    def forward(self, feats):
        running = {k: self.buf[k] for k in KM.running_names(self.cfg["backbone"])}
        sd = dict(self.buf, **dict(zip(self.names, self.params)))
        return KM.mdtc_train_logits(sd, self.cfg, feats, running)[0], None


def oracle_criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    return K.criterion(type, logits, target, lengths, target_lengths, min_duration, validation)


def test_executor_train_end_to_end():
    cfg, model, sd = shipped_model("mdtc_small")
    gpu = model.to(DEV).enable_training()
    cpu = OracleMdtc(cfg, sd)
    gen = torch.Generator().manual_seed(8)
    batches = []
    for _ in range(4):
        lens = torch.randint(30, 61, (8,), generator=gen)
        lens[0] = 60
        batches.append(dict(feats=torch.randn(8, 60, 80, generator=gen), target=torch.tensor([[0]] * 8),
                            feats_lengths=lens, target_lengths=torch.ones(8, dtype=torch.long)))
    args = {"criterion": "max_pooling", "grad_clip": 5.0}
    # one step with a zero learning rate: the gradients and the running statistics of the same weights
    for m, crit, d in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV)):
        KG.train(crit, m, torch.optim.SGD(m.parameters(), lr=0.0), batches[:1], torch.device(d), args)
    for n, p, q in zip(cpu.names, cpu.parameters(), gpu.parameters()):
        torch.testing.assert_close(q.grad.cpu(), p.grad, rtol=1e-3, atol=1e-5, msg=n)
    for k, v in cpu.buf.items():
        if "running" in k:
            torch.testing.assert_close(gpu.state_dict()[k].cpu(), v, rtol=1e-4, atol=1e-6, msg=k)
    # Adam steps: the losses follow (the weights themselves drift apart where a gradient is zero up to round-off, as
    # for the conv biases in front of a BatchNorm, which Adam moves by +-lr whatever the sign of the round-off)
    logs = [KG.train(crit, m, torch.optim.Adam(m.parameters(), lr=1e-3), batches, torch.device(d), args)
            for m, crit, d in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV))]
    for (a, sa), (b, sb) in zip(*logs):
        assert sa and sb and abs(a - b) <= 1e-3 * abs(a)


def test_determinism_no_grad_and_launch_counts():
    cfg, model, _ = shipped_model("mdtc")
    model = model.to(DEV).enable_training().train()
    L = 1 + 4 * 4
    gen = torch.Generator().manual_seed(4)
    feats = torch.randn(16, 150, 80, generator=gen).to(DEV)
    up = torch.randn(16, 150, 1, generator=gen).to(DEV)
    start = copy.deepcopy(model.state_dict())
    outs = []
    for _ in range(2):
        model.load_state_dict(start)
        model.zero_grad(set_to_none=True)
        n0 = _native.launch_count()
        y, _ = model(feats)
        torch.cuda.synchronize()
        fwd = _native.launch_count() - n0
        n0 = _native.launch_count()
        (y * up).sum().backward()
        torch.cuda.synchronize()
        bwd = _native.launch_count() - n0
        assert (fwd, bwd) == (2 + 3 * L, 3 + 4 * L)
        outs.append((y.detach().clone(), [p.grad.clone() for p in model.parameters()],
                     [t.clone() for t in running(model)]))
    (y1, g1, r1), (y2, g2, r2) = outs
    for a, b in zip([y1] + g1 + r1, [y2] + g2 + r2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    # no_grad: the same batch-statistics forward, bit for bit, with the forward's launches only and no saved buffer
    model.load_state_dict(start)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    with torch.no_grad():
        n0 = _native.launch_count()
        y3, _ = model(feats)
        torch.cuda.synchronize()
        assert _native.launch_count() - n0 == 2 + 3 * L
    assert not y3.requires_grad
    assert torch.equal(y3.view(torch.int32), y1.view(torch.int32))
    for a, b in zip(running(model), r1):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    saved_bytes = 4 * mdtc_train.saved_floats(L, 64, 16, 150)
    assert torch.cuda.max_memory_allocated(DEV) - base < saved_bytes / 2


def test_eval_after_a_training_step_repacks():
    cfg, model, _ = shipped_model("mdtc")
    model = model.to(DEV).enable_training()
    feats = torch.randn(4, 120, 80, device=DEV)
    with torch.no_grad():
        y_before, _ = model.eval()(feats)                       # packs the eval model
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    model.train()
    y, _ = model(feats)
    y.sum().backward()
    opt.step()
    with torch.no_grad():
        y_after, _ = model.eval()(feats)
    fresh = init_model(cfg)
    fresh.load_state_dict(model.state_dict())
    with torch.no_grad():
        y_fresh, _ = fresh.to(DEV).eval()(feats)
    assert torch.equal(y_after.view(torch.int32), y_fresh.view(torch.int32))
    assert not torch.equal(y_after, y_before)
    # a no_grad training forward changes only the running statistics: eval sees them too
    model.train()
    with torch.no_grad():
        model(feats * 2.0)
        y_stats, _ = model.eval()(feats)
    fresh.load_state_dict(model.state_dict())
    with torch.no_grad():
        y_fresh, _ = fresh.eval()(feats)
    assert torch.equal(y_stats.view(torch.int32), y_fresh.view(torch.int32))


def test_refusals_on_the_device():
    _, model, _ = shipped_model("mdtc_small")
    model = model.to(DEV).enable_training().train()
    feats = torch.randn(2, 10, 80, device=DEV)
    y, _ = model(feats)
    g = torch.autograd.grad(y.sum(), list(model.parameters()), create_graph=True)
    assert not any(t.requires_grad for t in g)            # once_differentiable: differentiating again is refused
    with pytest.raises(RuntimeError):
        g[0].sum().backward()
    conv = model.backbone.blocks[0].res_blocks[1].conv2
    w = conv.weight
    conv.weight = torch.nn.Parameter(w.detach().transpose(0, 1).contiguous().transpose(0, 1))
    assert not conv.weight.is_contiguous()
    with pytest.raises(ValueError, match="contiguous float32"):
        model(feats)
    conv.weight = torch.nn.Parameter(w.detach().double())
    with pytest.raises(ValueError, match="contiguous float32"):
        model(feats)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        model(torch.randn(1, 1, 80, device=DEV))
    with pytest.raises(RuntimeError, match="inference-only"):
        init_model(model_config("mdtc")).to(DEV).train()(feats)
