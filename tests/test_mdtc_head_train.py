"""Speech-command MDTC training (the `global` / `last` head) on the device: the head's Dropout mask hook against its
numpy restatement; logits, out_cache, running statistics and every parameter gradient against the reference's golden
cases and against the float64 oracle with the same mask; the recipe's shapes and edge shapes; p = 0 and p = 1;
determinism, the no_grad path, launch counts, eval after a step; Executor.train end to end."""
import copy

import numpy as np
import pytest
import torch

from oracle import kws_criterion_grad_oracle as KG
from oracle import kws_criterion_oracle as K
from oracle import kws_mdtc_head_train_oracle as KH
from oracle import kws_mdtc_train_oracle as KM
from tests.head_cases import head_config
from tests.test_mdtc_head_train_host import NAMES, golden, golden_call
from tests.test_mdtc_train_host import assert_within_rule
from wekws_b200 import _native, criterion, init_model, mdtc_train, synth
from wekws_b200.frontend import draw_seed

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FLOOR = 2.0 ** -20


def running(model):
    return [t for bn in mdtc_train.batch_norms(model) for t in (bn.running_mean, bn.running_var)]


def shipped(case, seed=5, **kw):
    """(cfg, model, state_dict) of a head case with synthetic weights; `kw` overrides config keys."""
    cfg = dict(head_config(case), **kw)
    torch.manual_seed(seed)
    model = synth.randomize_(init_model(cfg), seed=seed)
    return cfg, model, {k: v.clone() for k, v in model.state_dict().items()}


def seed_of(call_seed):
    """The Dropout seed a training forward draws after torch.manual_seed(call_seed)."""
    torch.manual_seed(call_seed)
    return draw_seed()


def train_step(model, feats, up, call_seed):
    model.enable_training(device_dropout=True).train()
    model.zero_grad(set_to_none=True)
    torch.manual_seed(call_seed)
    y, cache = model(feats)
    (y * up).sum().backward()
    return y.detach(), cache, [p.grad.detach().clone() for p in model.parameters()]


def oracle(sd, cfg, feats, up, p, call_seed, dtype):
    mask = None if p == 0 else KH.head_mask(seed_of(call_seed), feats.shape[0], p)
    return KH.mdtc_head_train_grads(sd, cfg, feats, up, mask, p, dtype, device=DEV)


def assert_rule(got, ref64, ref32, what, floor=FLOOR):
    """Each tensor: |value - float64| <= 8 x (torch float32's own error on the device) + floor x its largest value."""
    for i, (d, b, e) in enumerate(zip(got, ref64, ref32)):
        d, b, e = d.detach().double().to(DEV), b.detach().double().to(DEV), e.detach().double().to(DEV)
        assert d.shape == b.shape, f"{what}: tensor {i}: shape {tuple(d.shape)} != {tuple(b.shape)}"
        err = float((d - b).abs().max())
        bound = 8.0 * float((e - b).abs().max()) + floor * float(b.abs().max())
        assert err <= bound, f"{what}: tensor {i}: error {err:.3e} > bound {bound:.3e}"


def check_against_oracle(case, B, T, what, seed=5, call_seed=7, p=None, **kw):
    cfg, model, sd = shipped(case, seed=seed, **kw)
    if p is not None:
        mdtc_train.head_dropout(model).p = p
    p = mdtc_train.head_dropout(model).p
    gen = torch.Generator().manual_seed(B * 1000 + T)
    feats = torch.randn(B, T, cfg["input_dim"], generator=gen)
    up = torch.randn(B, cfg["output_dim"], generator=gen)
    model = model.to(DEV)
    y, cache, grads = train_step(model, feats.to(DEV), up.to(DEV), call_seed)
    y64, g64, r64, c64 = oracle(sd, cfg, feats, up, p, call_seed, torch.float64)
    y32, g32, r32, c32 = oracle(sd, cfg, feats, up, p, call_seed, torch.float32)
    rn = KM.running_names(cfg["backbone"])
    assert y.shape == (B, cfg["output_dim"]) and cache.shape == model.cache_shape(B)
    assert_rule(grads, g64, g32, what + " gradients")
    assert_rule(running(model), [r64[k] for k in rn], [r32[k] for k in rn], what + " running")
    assert_rule([y, cache], [y64, c64], [y32, c32], what + " logits / out_cache")
    return model, grads


def test_mask_hook_is_the_numpy_mask():
    for seed, B, p in ((0x0123456789ABCDEF, 100, 0.5), (7, 3, 0.1), (2 ** 63 + 5, 256, 0.9)):
        theta = int(np.ceil(p * 2.0 ** 24))
        out = torch.empty(B, 1, 64, dtype=torch.uint8, device=DEV)
        _native.call("wekws_dropout_mask", seed, B, 1, 64, 255, theta, out, device=DEV)
        assert np.array_equal(out.cpu().numpy()[:, 0, :].astype(bool), KH.head_mask(seed, B, p))


@pytest.mark.parametrize("name", NAMES)
def test_golden_cases(name):
    cfg, model, feats, mask, p = golden_call(name)
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    bb = cfg["backbone"]
    model = model.to(DEV)
    counts = [int(bn.num_batches_tracked) for bn in mdtc_train.batch_norms(model)]
    up = torch.from_numpy(golden(name, "up64")).float()
    y, _, grads = train_step(model, feats.to(DEV), up.to(DEV), int(golden(name, "call_seed")))
    assert [int(bn.num_batches_tracked) for bn in mdtc_train.batch_norms(model)] == [c + 1 for c in counts]
    y64, g64, r64, _ = KH.mdtc_head_train_grads(sd, cfg, feats, torch.from_numpy(golden(name, "up64")), mask, p,
                                                torch.float64)
    e_g, e_r = [float(e) for e in golden(name, "err32_g")], [float(e) for e in golden(name, "err32_run")]
    # the reference's own CPU float32 error as the unit, plus the project's floor of 2^-20 of each tensor's largest value
    fl = lambda ts, es: [e + FLOOR / 8 * float(t.abs().max()) for t, e in zip(ts, es)]
    assert_within_rule(grads, g64, fl(g64, e_g), name)
    rn = KM.running_names(bb)
    assert_within_rule(running(model), [r64[k] for k in rn], fl([r64[k] for k in rn], e_r), name)
    assert_within_rule([y], [y64], fl([y64], [float(golden(name, "err32_l"))]), name)


@pytest.mark.parametrize("case,B,T", [("mdtc_global", 100, 98), ("mdtc_last", 100, 98), ("mdtc_small_last", 64, 98)])
def test_recipe_shapes_against_oracle(case, B, T):
    check_against_oracle(case, B, T, f"{case} B={B} T={T}")


@pytest.mark.parametrize("case,B,T", [("mdtc_global", 8, 1), ("mdtc_last", 2, 1), ("mdtc_global", 4, 7),
                                      ("mdtc_small_last", 5, 11), ("mdtc_global", 1, 37), ("mdtc_last", 1, 5)])
def test_edge_shapes(case, B, T):
    """One frame per utterance (B rows of batch statistics); fewer frames than the model's padding; one utterance."""
    check_against_oracle(case, B, T, f"{case} B={B} T={T}")


def test_wide_output():
    check_against_oracle("mdtc_global", 6, 20, "odim 300", output_dim=300)


def test_p0_draws_no_seed_and_matches_no_dropout():
    cfg, model, sd = shipped("mdtc_global")
    mdtc_train.head_dropout(model).p = 0.0
    model = model.to(DEV).enable_training(device_dropout=True).train()
    feats = torch.randn(4, 30, 80)
    up = torch.randn(4, 11)
    torch.manual_seed(11)
    state = torch.get_rng_state()
    y, _ = model(feats.to(DEV))
    assert torch.equal(torch.get_rng_state(), state)            # nothing drawn
    (y * up.to(DEV)).sum().backward()
    grads = [p.grad for p in model.parameters()]
    y64, g64, _, _ = KH.mdtc_head_train_grads(sd, cfg, feats, up, None, 0.0, torch.float64, device=DEV)
    y32, g32, _, _ = KH.mdtc_head_train_grads(sd, cfg, feats, up, None, 0.0, torch.float32, device=DEV)
    assert_rule(grads + [y], g64 + [y64], g32 + [y32], "p = 0")


def test_p1_gives_exact_zeros():
    model, grads = check_against_oracle("mdtc_last", 8, 20, "p = 1", p=1.0)
    names = [n for n, _ in model.named_parameters()]
    for n, g in zip(names, grads):
        if n != "classifier.classifier.3.bias":
            assert not bool(g.any()), n


def test_determinism_no_grad_and_launch_counts():
    cfg, model, _ = shipped("mdtc_global")
    model = model.to(DEV).enable_training(device_dropout=True).train()
    L = 17
    gen = torch.Generator().manual_seed(4)
    feats = torch.randn(32, 98, 80, generator=gen).to(DEV)
    up = torch.randn(32, 11, generator=gen).to(DEV)
    start = copy.deepcopy(model.state_dict())
    outs = []
    for _ in range(2):
        model.load_state_dict(start)
        model.zero_grad(set_to_none=True)
        torch.manual_seed(9)
        n0 = _native.launch_count()
        y, _ = model(feats)
        torch.cuda.synchronize()
        fwd = _native.launch_count() - n0
        n0 = _native.launch_count()
        (y * up).sum().backward()
        torch.cuda.synchronize()
        bwd = _native.launch_count() - n0
        assert (fwd, bwd) == (mdtc_train.head_forward_launches(L), mdtc_train.head_backward_launches(L)) \
            == (3 + 3 * L, 4 + 4 * L)
        outs.append((y.detach().clone(), [p.grad.clone() for p in model.parameters()],
                     [t.clone() for t in running(model)]))
    (y1, g1, r1), (y2, g2, r2) = outs
    for a, b in zip([y1] + g1 + r1, [y2] + g2 + r2):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    torch.manual_seed(10)                                        # another seed: another mask
    model.load_state_dict(start)
    y_other, _ = model(feats)
    assert not torch.equal(y_other, y1)
    # no_grad: the same forward bit for bit (same seed), the forward's launches only, no saved buffer
    model.load_state_dict(start)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    with torch.no_grad():
        torch.manual_seed(9)
        n0 = _native.launch_count()
        y3, _ = model(feats)
        torch.cuda.synchronize()
        assert _native.launch_count() - n0 == 3 + 3 * L
    assert not y3.requires_grad
    assert torch.equal(y3.view(torch.int32), y1.view(torch.int32))
    for a, b in zip(running(model), r1):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.cuda.max_memory_allocated(DEV) - base < 4 * mdtc_train.head_saved_floats(L, 64, 32, 98) / 2


def test_eval_after_a_training_step_repacks():
    cfg, model, _ = shipped("mdtc_global")
    model = model.to(DEV).enable_training(device_dropout=True)
    feats = torch.randn(4, 98, 80, device=DEV)
    with torch.no_grad():
        y_before, _ = model.eval()(feats)
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
    assert y_after.shape == (4, 11)
    assert torch.equal(y_after.view(torch.int32), y_fresh.view(torch.int32))
    assert not torch.equal(y_after, y_before)


class OracleHead(torch.nn.Module):
    """The oracle's training forward as a torch model with the same parameters, in the same order, drawing its mask's
    seed from torch's generator as the device model does."""

    def __init__(self, cfg, sd, p):
        super().__init__()
        self.cfg, self.names, self.p = cfg, KH.param_names(cfg["backbone"]), p
        self.params = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone()) for n in self.names])
        self.buf = {k: v.clone() for k, v in sd.items() if k not in self.names}

    def forward(self, feats):
        running = {k: self.buf[k] for k in KM.running_names(self.cfg["backbone"])}
        sd = dict(self.buf, **dict(zip(self.names, self.params)))
        mask = KH.head_mask(draw_seed(), feats.shape[0], self.p) if self.p > 0 else None
        return KH.mdtc_head_train_logits(sd, self.cfg, feats, running, mask, self.p)[0], None


def oracle_criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    return K.criterion(type, logits, target, lengths, target_lengths, min_duration, validation)


def test_executor_train_end_to_end():
    cfg, model, sd = shipped("mdtc_global")
    gpu = model.to(DEV).enable_training(device_dropout=True)
    cpu = OracleHead(cfg, sd, mdtc_train.head_dropout(model).p)
    gen = torch.Generator().manual_seed(8)
    batches = [dict(feats=torch.randn(16, 98, 80, generator=gen), target=torch.randint(0, 11, (16, 1), generator=gen),
                    feats_lengths=torch.full((16,), 98), target_lengths=torch.ones(16, dtype=torch.long))
               for _ in range(4)]
    args = {"criterion": "ce", "grad_clip": 5.0}
    # one step with a zero learning rate: the gradients and the running statistics of the same weights and mask
    for m, crit, d in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV)):
        torch.manual_seed(31)
        KG.train(crit, m, torch.optim.SGD(m.parameters(), lr=0.0), batches[:1], torch.device(d), args)
    for n, p, q in zip(cpu.names, cpu.parameters(), gpu.parameters()):
        torch.testing.assert_close(q.grad.cpu(), p.grad, rtol=1e-3, atol=1e-5, msg=n)
    for k, v in cpu.buf.items():
        if "running" in k:
            torch.testing.assert_close(gpu.state_dict()[k].cpu(), v, rtol=1e-4, atol=1e-6, msg=k)
    # Adam steps, each drawing its own mask from the same generator state: the losses follow
    logs = []
    for m, crit, d in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV)):
        torch.manual_seed(32)
        logs.append(KG.train(crit, m, torch.optim.Adam(m.parameters(), lr=1e-3), batches, torch.device(d), args))
    for (a, sa), (b, sb) in zip(*logs):
        assert sa and sb and abs(a - b) <= 1e-3 * abs(a)
