"""GRU training on the device: training-mode logits against the eval kernel's, parameter gradients against the
reference's (golden) and the float64 oracle's, every streams-per-CTA partition of the forward and the backward,
Executor.train end to end, determinism, launch counts and refusals."""
import pytest
import torch

from oracle import kws_criterion_grad_oracle as KC
from oracle import kws_criterion_oracle as K
from oracle import kws_gru_train_oracle as KG
from tests.test_gru_train_host import NAMES, assert_within_rule, golden, golden_feats, golden_model
from wekws_b200 import _native, criterion, init_model, model_config, synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def device_model(case):
    """(cfg, CPU state_dict, GRU model on the device opted in to training) of a golden case."""
    cfg, model = golden_model(case)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    return cfg, sd, model.to(DEV).enable_training(bptt=True)


def train_step(model, feats, up):
    """Training-mode forward and backward of (logits * up).sum(); returns (logits, out_cache, grads)."""
    model.train()
    model.zero_grad(set_to_none=True)
    y, cache = model(feats)
    assert y.requires_grad and not cache.requires_grad
    (y * up).sum().backward()
    return y.detach(), cache, [p.grad.detach().clone() for p in model.parameters()]


def eval_fp32(model, feats):
    model.eval()
    model.precision = "fp32"
    try:
        with torch.no_grad():
            return model(feats)
    finally:
        model.precision = "auto"


def oracle_check(cfg, sd, feats, up, grads, what):
    """The gradients against the float64 oracle under the rule, with the oracle's own float32 error as the noise."""
    _, g32 = KG.gru_grads(sd, cfg, feats, up, torch.float32)
    _, g64 = KG.gru_grads(sd, cfg, feats, up, torch.float64)
    err32 = [float((a.double() - b).abs().max()) for a, b in zip(g32, g64)]
    assert_within_rule(grads, g64, err32, what)


@pytest.mark.parametrize("name", NAMES)
def test_golden_logits_and_gradients(name):
    cfg, sd, model = device_model(str(golden(name, "case")))
    feats = golden_feats(name, cfg)
    up64 = torch.from_numpy(golden(name, "up64"))
    y, cache, grads = train_step(model, feats.to(DEV), up64.float().to(DEV))
    ref = torch.from_numpy(golden(name, "logits"))
    torch.testing.assert_close(y.cpu(), ref, rtol=1e-4, atol=1e-4 * float(ref.abs().max()))
    y_eval, cache_eval = eval_fp32(model, feats.to(DEV))
    assert torch.equal(y.view(torch.int32), y_eval.view(torch.int32))       # the FP32 eval logits, bit for bit
    assert torch.equal(cache.view(torch.int32), cache_eval.view(torch.int32))
    # the float64 gradients whose digests the reference pinned (tests/test_gru_train_host.py)
    _, g64 = KG.gru_grads(sd, cfg, feats, up64, torch.float64)
    assert_within_rule(grads, g64, [float(e) for e in golden(name, "err32_g")], name)


def shipped(seed=3):
    """gru.yaml (input_dim 40, output_dim 2, global CMVN) with synthetic weights: (cfg, CPU state_dict, model)."""
    cfg, model = KG.golden_model("gru", init_model, seed=seed)
    return cfg, {k: v.clone() for k, v in model.state_dict().items()}, model.to(DEV).enable_training(bptt=True)


def test_shipped_batch_against_oracle():
    cfg, sd, model = shipped()
    gen = torch.Generator().manual_seed(2)
    feats = synth.features(256, 50, 40, seed=5, cmvn_like=True)
    up = torch.randn(256, 50, 2, generator=gen)
    up[7, 30:] = 0.0                                                          # padding rows
    y, cache, grads = train_step(model, feats.to(DEV), up.to(DEV))
    y_eval, cache_eval = eval_fp32(model, feats.to(DEV))
    assert torch.equal(y.view(torch.int32), y_eval.view(torch.int32))
    assert torch.equal(cache.view(torch.int32), cache_eval.view(torch.int32))
    oracle_check(cfg, sd, feats, up, grads, "shipped B=256")


def test_every_streams_per_cta_partition():
    """Batches from the SM count that select S = 1, 2, 4 and 8 streams per CTA in the forward and the backward, with
    a partial last tile; every stream's logits and cache against the float64 oracle, the gradients under the rule."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    cfg, sd, model = shipped(seed=4)
    for B, S in ((sms - 1, 1), (2 * sms - 1, 2), (3 * sms + 1, 4), (4 * sms + 3, 8)):
        gen = torch.Generator().manual_seed(B)
        feats = synth.features(B, 6, 40, seed=B, cmvn_like=True)
        up = torch.randn(B, 6, 2, generator=gen)
        y, cache, grads = train_step(model, feats.to(DEV), up.to(DEV))
        y64, c64 = KG.gru_logits({k: v.double() for k, v in sd.items()}, cfg, feats.double())
        err = (y.cpu().double() - y64).abs().amax(dim=(1, 2))
        assert float(err.max()) <= 1e-5, f"B={B} (S={S}): stream {int(err.argmax())} off by {float(err.max()):.2e}"
        cerr = (cache.cpu().double() - c64).abs().amax(dim=(0, 2))
        assert float(cerr.max()) <= 1e-5, f"B={B} (S={S}): cache of stream {int(cerr.argmax())}"
        oracle_check(cfg, sd, feats, up, grads, f"B={B} (S={S})")


@pytest.mark.parametrize("B,T", [(1, 1), (0, 5), (3, 0)])
def test_edge_shapes(B, T):
    cfg, sd, model = device_model("gru")
    feats = synth.features(B, T, 40, seed=9, cmvn_like=True)
    up = torch.randn(B, T, 2)
    y, cache, grads = train_step(model, feats.to(DEV), up.to(DEV))
    assert y.shape == (B, T, 2) and cache.shape == (2, B, 128)
    if B * T == 0:
        assert all(float(g.abs().max()) == 0.0 for g in grads)
    else:
        oracle_check(cfg, sd, feats, up, grads, f"B={B} T={T}")


def test_backward_is_deterministic():
    _, _, model = shipped()
    model.train()
    feats = synth.features(64, 80, 40, seed=6, cmvn_like=True).to(DEV)
    up = torch.randn(64, 80, 2, generator=torch.Generator().manual_seed(6)).to(DEV)
    y, _ = model(feats)
    loss = (y * up).sum()
    g1 = torch.autograd.grad(loss, list(model.parameters()), retain_graph=True)
    g2 = torch.autograd.grad(loss, list(model.parameters()))
    for a, b in zip(g1, g2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


class OracleGru(torch.nn.Module):
    """The oracle's GRU model forward as a torch model with the same parameters, in the same order."""

    def __init__(self, cfg, sd):
        super().__init__()
        self.cfg, self.names = cfg, KG.param_names(cfg["backbone"]["num_layers"])
        self.params = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone()) for n in self.names])
        self.buf = {k: v.clone() for k, v in sd.items() if k not in self.names}

    def forward(self, feats):
        return KG.gru_logits(dict(self.buf, **dict(zip(self.names, self.params))), self.cfg, feats)


def oracle_criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    return K.criterion(type, logits, target, lengths, target_lengths, min_duration, validation)


def test_executor_train_end_to_end():
    cfg, sd, gpu = device_model("gru")
    cpu = OracleGru(cfg, sd)
    gen = torch.Generator().manual_seed(8)
    batches = []
    for _ in range(5):
        lens = torch.randint(12, 31, (8,), generator=gen)
        lens[0] = 30
        batches.append(dict(feats=torch.randn(8, 30, 40, generator=gen) * 3 + 15,
                            target=torch.randint(-1, 2, (8, 1), generator=gen), feats_lengths=lens,
                            target_lengths=torch.ones(8, dtype=torch.long)))
    args = {"criterion": "max_pooling", "grad_clip": 5.0}
    for model, crit, device in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV)):
        KC.train(crit, model, torch.optim.SGD(model.parameters(), lr=0.0), batches[:1], torch.device(device), args)
    for n, p, q in zip(cpu.names, cpu.parameters(), gpu.parameters()):
        assert torch.allclose(q.grad.cpu(), p.grad, rtol=1e-4, atol=1e-6), n
    logs = [KC.train(crit, model, torch.optim.Adam(model.parameters(), lr=1e-3), batches, torch.device(device), args)
            for model, crit, device in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV))]
    assert [s for _, s in logs[0]] == [s for _, s in logs[1]] == [True] * 5
    for (a, _), (b, _) in zip(*logs):
        assert abs(a - b) <= 1e-3 * abs(a)
    # after training, eval repacks from the host (the version counters moved): eval == oracle on the trained weights
    with torch.no_grad():
        y, _ = gpu.eval()(batches[0]["feats"].to(DEV))
        y_ref = cpu(batches[0]["feats"])[0]
    torch.testing.assert_close(y.cpu(), y_ref, rtol=1e-4, atol=1e-5)


def test_launch_counts_and_no_grad_path():
    cfg, _, model = device_model("gru_l4_id37")
    L = cfg["backbone"]["num_layers"]
    for B, T in ((3, 5), (300, 40)):
        feats = torch.randn(B, T, 80, device=DEV)
        model.precision = "fp32"
        with torch.no_grad():
            y_eval, _ = model.eval()(feats)
            n0 = _native.launch_count()
            y_nograd, _ = model.train()(feats)                                 # training mode without grad: eval
            torch.cuda.synchronize()
            assert _native.launch_count() - n0 == 1
            assert torch.equal(y_nograd.view(torch.int32), y_eval.view(torch.int32)) and not y_nograd.requires_grad
        model.precision = "tensor"                       # the training forward runs the FP32 kernel regardless
        n0 = _native.launch_count()
        y, _ = model(feats)
        torch.cuda.synchronize()
        assert _native.launch_count() - n0 == 2                                # pack + the storing forward
        assert torch.equal(y.detach().view(torch.int32), y_eval.view(torch.int32))
        n0 = _native.launch_count()
        y.sum().backward()
        torch.cuda.synchronize()
        assert _native.launch_count() - n0 == 5 + 4 * L
        model.precision = "auto"


def test_refusals():
    _, _, model = device_model("gru")
    model.train()
    feats = torch.randn(2, 10, 40, device=DEV)
    _, cache = model(feats)
    with pytest.raises(ValueError, match="streaming cache"):
        model(feats, cache)
    with pytest.raises(ValueError, match="features that require grad"):
        model(feats.clone().requires_grad_(True))
    with pytest.raises(RuntimeError, match="forward_softmax has no training path"):
        model.forward_softmax(feats)
    y, _ = model(feats)
    g = torch.autograd.grad(y.sum(), list(model.parameters()), create_graph=True)
    assert not any(t.requires_grad for t in g)           # once_differentiable: the gradients are constants,
    with pytest.raises(RuntimeError):                    # so differentiating them again is refused
        g[0].sum().backward()
    w = model.classifier.linear.weight
    model.classifier.linear.weight = torch.nn.Parameter(w.detach().t().contiguous().t())
    with pytest.raises(ValueError, match="contiguous float32"):
        model(feats)
    model.classifier.linear.weight = torch.nn.Parameter(w.detach().double())
    with pytest.raises(ValueError, match="contiguous float32"):
        model(feats)
    other = init_model(model_config("gru")).to(DEV).train()
    with pytest.raises(RuntimeError, match="inference-only"):
        other(torch.randn(1, 8, 80, device=DEV))
