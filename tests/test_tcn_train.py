"""TCN / DS-TCN training on the device: the Dropout mask hook against its numpy restatement; logits, running
statistics and parameter gradients against the reference's golden cases and against the float64 oracle with the same
masks across hidden sizes, both backbones, CMVN, kernel sizes and layer counts; Executor.train end to end; determinism,
the p = 0 and no_grad paths, eval after a step, launch counts and edge shapes."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import kws_criterion_grad_oracle as KG
from oracle import kws_criterion_oracle as K
from oracle import kws_tcn_train_oracle as KT
from tests.test_mdtc_train_host import assert_within_rule
from tests.test_tcn_train_host import NAMES, golden, golden_feats, golden_masks, golden_model
from wekws_b200 import _native, criterion, init_model, model_config, synth, tcn_train
from wekws_b200.frontend import draw_seed

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
FLOOR = 2.0 ** -20


def running(model):
    return [t for bn in tcn_train.batch_norms(model) for t in (bn.running_mean, bn.running_var)]


def shipped(name, hidden=None, K=None, L=None, norm_var=None, **kw):
    """(cfg, model, state_dict) of a recipe model, with hidden_dim / kernel_size / num_layers overridden and a global
    CMVN (norm_var True or False) when asked."""
    path = synth.write_cmvn_json(kw.get("input_dim", 80)) if norm_var is not None else None
    cfg = model_config(name, cmvn_file=path, norm_var=bool(norm_var), **kw)
    if hidden is not None:
        cfg["hidden_dim"] = hidden
    if K is not None:
        cfg["backbone"]["kernel_size"] = K
    if L is not None:
        cfg["backbone"]["num_layers"] = L
    try:
        torch.manual_seed(5)
        model = synth.randomize_(init_model(cfg), seed=5)
    finally:
        if path:
            os.unlink(path)
            cfg["cmvn"] = dict(norm_var=norm_var)
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


def oracle(sd, cfg, feats, up, ps, call_seed, dtype):
    B, T = feats.shape[0], feats.shape[1]
    masks = None if all(p == 0 for p in ps) else KT.dropout_masks(seed_of(call_seed), B, T, cfg["hidden_dim"], ps)
    return KT.tcn_train_grads(sd, cfg, feats, up, masks, ps, dtype, device=DEV)


def assert_rule(got, ref64, ref32, what, floor=FLOOR):
    """Each tensor: |value - float64| <= 8 x (torch float32's own error on the device) + floor x its largest value."""
    for i, (d, b, e) in enumerate(zip(got, ref64, ref32)):
        d, b, e = d.detach().double().to(DEV), b.detach().double().to(DEV), e.detach().double().to(DEV)
        assert d.shape == b.shape, f"{what}: tensor {i}: shape {tuple(d.shape)} != {tuple(b.shape)}"
        err = float((d - b).abs().max())
        bound = 8.0 * float((e - b).abs().max()) + floor * float(b.abs().max())
        assert err <= bound, f"{what}: tensor {i}: error {err:.3e} > bound {bound:.3e}"


def check_against_oracle(name, B, T, what, floor=FLOOR, **kw):
    cfg, model, sd = shipped(name, **kw)
    ps = [d.p for d in tcn_train.dropouts(model)]
    model = model.to(DEV)
    gen = torch.Generator().manual_seed(B * 1000 + T)
    feats = torch.randn(B, T, cfg["input_dim"], generator=gen)
    if "cmvn" in cfg:
        feats = feats * 3.0 + 15.0                         # log-mel-like, as the CMVN expects
    up = torch.randn(B, T, cfg["output_dim"], generator=gen)
    tf32 = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        y64, g64, r64, c64 = oracle(sd, cfg, feats, up, ps, 11, torch.float64)
        y32, g32, r32, c32 = oracle(sd, cfg, feats, up, ps, 11, torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf32
    y, cache, grads = train_step(model, feats.to(DEV), up.to(DEV), 11)
    rn = KT.running_names(cfg["backbone"])
    assert_rule(grads, g64, g32, what + " gradients", floor)
    assert_rule(running(model), [r64[k] for k in rn], [r32[k] for k in rn], what + " running", floor)
    assert_rule([y], [y64], [y32], what + " logits", floor)
    assert_rule([cache], [c64], [c32], what + " out_cache", floor)


def test_dropout_mask_hook_matches_numpy():
    for seed, B, T, C, layer, p in ((0x123456789ABCDEF0, 3, 7, 64, 0, 0.1), (2 ** 64 - 1, 2, 5, 256, 3, 0.5),
                                    (42, 1, 1, 64, 7, 0.0), (42, 2, 3, 64, 1, 1.0)):
        out = torch.empty(B, T, C, dtype=torch.uint8, device=DEV)
        _native.call("wekws_dropout_mask", seed, B, T, C, layer, KT.theta(p), out, device=DEV)
        want = KT.dropout_mask(seed, B, T, C, layer, p)
        assert np.array_equal(out.cpu().numpy().astype(bool), want), (seed, layer, p)


def test_keep_fraction():
    B, T, C = 250, 200, 256                                   # 1.28e7 elements
    for p in (0.1, 0.5, 0.9):
        out = torch.empty(B, T, C, dtype=torch.uint8, device=DEV)
        _native.call("wekws_dropout_mask", 77, B, T, C, 2, KT.theta(p), out, device=DEV)
        n = out.numel()
        q = 1.0 - KT.theta(p) / 2.0 ** 24
        frac = float(out.double().mean())
        assert abs(frac - q) <= 5.0 * math.sqrt(q * (1 - q) / n), (p, frac, q)


@pytest.mark.parametrize("name,B,T,kw", [("ds_tcn", 4, 60, {}), ("tcn", 3, 50, {}),
                                         ("ds_tcn", 2, 40, dict(activation="identity", output_dim=37, input_dim=40)),
                                         ("tcn", 2, 30, dict(activation="identity", output_dim=2599))])
def test_small_cases_against_oracle(name, B, T, kw):
    check_against_oracle(name, B, T, f"{name} B={B} T={T}", **kw)


@pytest.mark.parametrize("name", NAMES)
def test_golden_cases(name):
    """The reference's own float32 error of float64 as the unit (the MDTC rule): 8x it plus 2^-24."""
    cfg, model = golden_model(str(golden(name, "case")))
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    feats = golden_feats(name, cfg)
    masks, ps = golden_masks(name, model)
    up64 = torch.from_numpy(golden(name, "up64"))
    y64, g64, r64, _ = KT.tcn_train_grads(sd, cfg, feats, up64, masks, ps, torch.float64)
    model = model.to(DEV)
    counts = [int(bn.num_batches_tracked) for bn in tcn_train.batch_norms(model)]
    y, _, grads = train_step(model, feats.to(DEV), up64.float().to(DEV), int(golden(name, "call_seed")))
    assert [int(bn.num_batches_tracked) for bn in tcn_train.batch_norms(model)] == [c + 1 for c in counts]
    rn = KT.running_names(cfg["backbone"])
    assert_within_rule(grads, g64, [float(e) for e in golden(name, "err32_g")], name + " gradients")
    assert_within_rule(running(model), [r64[k] for k in rn], [float(e) for e in golden(name, "err32_run")],
                       name + " running")
    assert_within_rule([y], [y64], [float(golden(name, "err32_l"))], name + " logits")


@pytest.mark.parametrize("name,B,T,kw", [
    ("ds_tcn", 4, 60, dict(hidden=64)),                                    # hey_snips ds_tcn.yaml
    ("tcn", 3, 40, dict(hidden=256)),
    ("ds_tcn", 3, 50, dict(hidden=64, norm_var=True, input_dim=40)),
    ("ds_tcn", 3, 50, dict(norm_var=False, input_dim=40)),
    ("tcn", 3, 50, dict(norm_var=False)),
    ("tcn", 4, 30, dict(K=3, L=2)),
    ("tcn", 2, 25, dict(K=2, L=1, hidden=256)),
    ("ds_tcn", 2, 300, dict(K=5, L=8, hidden=64)),                         # pad_total 1020, T < the last padding
    ("ds_tcn", 2, 40, dict(K=4, L=8, hidden=256, output_dim=5)),
])
def test_configurations_against_oracle(name, B, T, kw):
    check_against_oracle(name, B, T, f"{name} {kw} B={B} T={T}", **kw)


@pytest.mark.parametrize("name,B,T", [("ds_tcn", 100, 200), ("tcn", 100, 200)])
def test_shipped_sizes_against_oracle(name, B, T):
    check_against_oracle(name, B, T, f"{name} shipped")


# B = 1, T = 2 (two rows of batch statistics) is left out.  Every BatchNorm's x_hat is then +-1 and its variance the
# square of one difference of two rows, so each float32 error is a few roundings amplified by 1 / |difference|, and
# torch's own float32 error is no stable unit at this shape: for ds_tcn (H100, these weights and inputs) the largest
# tap-gradient error of torch float32 is 6.4e-4 on CUDA but 2.6e-2 on the CPU, 40x apart.  The device's 9.2e-3 is
# 1.8x the 8x-CUDA bound and a third of torch's CPU error.  B = 2, T = 1 keeps a two-row batch in the list.
@pytest.mark.parametrize("B,T", [(1, 3), (2, 1), (3, 5), (1, 130), (5, 77)])
def test_edge_shapes(B, T):
    check_against_oracle("ds_tcn", B, T, f"ds_tcn B={B} T={T}")
    check_against_oracle("tcn", B, T, f"tcn B={B} T={T}")


def test_determinism_seed_and_no_grad():
    cfg, model, sd = shipped("ds_tcn")
    model = model.to(DEV).enable_training(device_dropout=True).train()
    feats = torch.randn(4, 50, 80, generator=torch.Generator().manual_seed(1)).to(DEV)
    up = torch.randn(4, 50, 1, generator=torch.Generator().manual_seed(2)).to(DEV)

    def run(seed):
        model.load_state_dict(sd)
        y, _, g = train_step(model, feats, up, seed)
        return y, g, [t.clone() for t in running(model)]

    a, b, c = run(3), run(3), run(4)
    for x, z in zip([a[0]] + a[1] + a[2], [b[0]] + b[1] + b[2]):
        assert torch.equal(x, z)
    assert not torch.equal(a[0], c[0])
    # the no_grad training forward: the same bits, the same running statistics, no saved buffer
    model.load_state_dict(sd)
    torch.manual_seed(3)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    before = torch.cuda.memory_allocated(DEV)
    with torch.no_grad():
        y, _ = model(feats)
    torch.cuda.synchronize()
    assert torch.equal(y, a[0]) and y.grad_fn is None
    assert all(torch.equal(x, z) for x, z in zip(running(model), a[2]))
    assert torch.cuda.max_memory_allocated(DEV) - before < tcn_train.saved_floats(4, 256, True, 4, 50) * 4


def test_p_zero_draws_nothing_and_matches_no_dropout():
    """p = 0 draws no seed and runs without a mask (theta 0 keeps every element, scale 1.0f is exact): checked
    against the oracle without Dropout within tolerance, and bitwise across generator states."""
    cfg, model, sd = shipped("tcn")
    for d in tcn_train.dropouts(model):
        d.p = 0.0
    model = model.to(DEV)
    feats = torch.randn(3, 40, 80, generator=torch.Generator().manual_seed(3))
    up = torch.randn(3, 40, 1, generator=torch.Generator().manual_seed(4))
    torch.manual_seed(9)
    state = torch.get_rng_state()
    model.enable_training(device_dropout=True).train()
    y, _ = model(feats.to(DEV))
    assert torch.equal(torch.get_rng_state(), state)           # nothing drawn
    (y * up.to(DEV)).sum().backward()
    y64, g64, _, _ = KT.tcn_train_grads(sd, cfg, feats, up, None, [0.0] * 4, torch.float64, device=DEV)
    y32, g32, _, _ = KT.tcn_train_grads(sd, cfg, feats, up, None, [0.0] * 4, torch.float32, device=DEV)
    assert_rule([y] + [p.grad for p in model.parameters()], [y64] + g64, [y32] + g32, "p = 0")
    torch.manual_seed(123)                                       # another generator state: the same bits
    model.load_state_dict(sd)
    y2, _ = model(feats.to(DEV))
    model.load_state_dict(sd)
    torch.manual_seed(9)
    y3, _ = model(feats.to(DEV))
    assert torch.equal(y2, y3)


def test_eval_after_a_training_step_repacks():
    cfg, model, sd = shipped("ds_tcn")
    model = model.to(DEV)
    feats = torch.randn(2, 30, 80, generator=torch.Generator().manual_seed(5)).to(DEV)
    y0, _ = model.eval()(feats)
    model.enable_training(device_dropout=True).train()
    opt = torch.optim.SGD(model.parameters(), lr=0.1)
    y, _ = model(feats)
    y.sum().backward()
    opt.step()
    y1, _ = model.eval()(feats)
    fresh = init_model(cfg).to(DEV).eval()
    fresh.load_state_dict(model.state_dict())
    y2, _ = fresh(feats)
    assert not torch.equal(y0, y1) and torch.equal(y1, y2)


@pytest.mark.parametrize("name", ["tcn", "ds_tcn"])
def test_launch_counts(name):
    cfg, model, sd = shipped(name)
    model = model.to(DEV).enable_training(device_dropout=True).train()
    L, ds = cfg["backbone"]["num_layers"], cfg["backbone"]["ds"]
    feats = torch.randn(2, 20, 80, device=DEV)
    n0 = _native.launch_count()
    y, _ = model(feats)
    assert _native.launch_count() - n0 == tcn_train.forward_launches(L, ds)
    n0 = _native.launch_count()
    y.sum().backward()
    assert _native.launch_count() - n0 == tcn_train.backward_launches(L, ds)
    n0 = _native.launch_count()
    with torch.no_grad():
        model(feats)
    assert _native.launch_count() - n0 == tcn_train.forward_launches(L, ds)


class OracleTcn(torch.nn.Module):
    """The oracle's training forward as a torch model with the same parameters, drawing its Dropout seed from torch's
    generator as the device model does."""

    def __init__(self, cfg, sd, ps, device):
        super().__init__()
        self.cfg, self.names, self.ps = cfg, KT.param_names(cfg["backbone"]), ps
        self.params = torch.nn.ParameterList([torch.nn.Parameter(sd[n].clone().to(device)) for n in self.names])
        self.buf = {k: v.clone().to(device) for k, v in sd.items() if k not in self.names}

    def forward(self, feats):
        B, T = feats.shape[0], feats.shape[1]
        masks = None
        if any(p > 0 for p in self.ps):
            masks = [torch.from_numpy(m) for m in KT.dropout_masks(draw_seed(), B, T, self.cfg["hidden_dim"], self.ps)]
        running = {k: self.buf[k] for k in KT.running_names(self.cfg["backbone"])}
        sd = dict(self.buf, **dict(zip(self.names, self.params)))
        return KT.tcn_train_logits(sd, self.cfg, feats, running, masks, self.ps)[0], None


def oracle_criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    return K.criterion(type, logits, target, lengths, target_lengths, min_duration, validation)


@pytest.mark.parametrize("case", ["tcn_max_pooling", "ds_tcn_ctc_2599"])
def test_executor_train_end_to_end(case):
    """Executor.train with the device criterion against the oracle model with the oracle criterion, the generator
    replayed so both draw the same Dropout seeds: the gradients and running statistics after one lr = 0 step, then
    the losses over Adam steps."""
    if case == "tcn_max_pooling":
        cfg, model, sd = shipped("tcn")
        idim, B, T, V = 80, 8, 60, None
    else:
        cfg, model, sd = shipped("ds_tcn", activation="identity", output_dim=2599)   # ds_tcn_ctc.yaml
        idim, B, T, V = 80, 6, 60, 2599
    ps = [d.p for d in tcn_train.dropouts(model)]
    gpu = model.to(DEV).enable_training(device_dropout=True)
    cpu = OracleTcn(cfg, sd, ps, "cpu")
    gen = torch.Generator().manual_seed(8)
    batches = []
    for _ in range(4):
        lens = torch.randint(30, T + 1, (B,), generator=gen)
        lens[0] = T
        if V is None:
            batches.append(dict(feats=torch.randn(B, T, idim, generator=gen), target=torch.tensor([[0]] * B),
                                feats_lengths=lens, target_lengths=torch.ones(B, dtype=torch.long)))
        else:
            batches.append(dict(feats=torch.randn(B, T, idim, generator=gen),
                                target=torch.randint(1, V, (B, 4), generator=gen), feats_lengths=lens,
                                target_lengths=torch.randint(1, 5, (B,), generator=gen)))
    args = {"criterion": "max_pooling" if V is None else "ctc", "grad_clip": 5.0}
    runs = ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV))
    for m, crit, d in runs:
        torch.manual_seed(21)
        KG.train(crit, m, torch.optim.SGD(m.parameters(), lr=0.0), batches[:1], torch.device(d), args)
    for n, p, q in zip(cpu.names, cpu.parameters(), gpu.parameters()):
        torch.testing.assert_close(q.grad.cpu(), p.grad, rtol=1e-3, atol=max(1e-5, 1e-4 * float(p.grad.abs().max())),
                                   msg=n)
    for k, v in cpu.buf.items():
        if "running" in k:
            torch.testing.assert_close(gpu.state_dict()[k].cpu(), v, rtol=1e-4, atol=1e-6, msg=k)
    logs = []
    for m, crit, d in runs:
        torch.manual_seed(22)
        logs.append(KG.train(crit, m, torch.optim.Adam(m.parameters(), lr=1e-3), batches, torch.device(d), args))
    for (a, sa), (b, sb) in zip(*logs):
        assert sa and sb and abs(a - b) <= 1e-3 * abs(a), (a, b)
