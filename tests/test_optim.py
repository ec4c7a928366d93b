"""The device optimiser (wekws_b200.Adam, wekws_b200.clip_grad_norm_) on the parameter sets of every shipped training
model, against torch.optim.Adam (foreach) and torch.nn.utils.clip_grad_norm_: one step against float64, 100-step
trajectories, edge cases, the clip's norm and non-finite paths, determinism, launch counts, version counters, the
state_dict round trip and Executor.train end to end."""
import copy
import math

import pytest
import torch

from tests.head_cases import head_config
from tests.test_optim_host import PARAM_SETS
from wekws_b200 import Adam, _native, clip_grad_norm_, criterion, init_model, model_config, synth

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# ours may be at most this many times torch float32's own largest error against float64 (+ one ulp of the value)
ADAM_ERR_FACTOR = 2.0


def params_of(name, seed=0):
    model = synth.randomize_(init_model(PARAM_SETS[name]()), seed=seed)
    return [p.detach().to(DEV) for p in model.parameters()]


def make_pair(base, **kw):
    """Two parameter lists with the same values, one for each optimiser."""
    a = [torch.nn.Parameter(t.clone()) for t in base]
    b = [torch.nn.Parameter(t.clone()) for t in base]
    return a, b, Adam(a, **kw), torch.optim.Adam(b, foreach=True, **kw)


def synth_grads(base, gen, scale=1e-2):
    return [(torch.randn(t.shape, generator=gen) * scale).to(DEV) for t in base]


def ordered(x):
    """float32 bits as integers that order like the values (ulp distance = difference)."""
    i = x.contiguous().view(torch.int32).to(torch.int64)
    return torch.where(i < 0, -(i & 0x7FFFFFFF), i)


def ulps(a, b):
    return int((ordered(a) - ordered(b)).abs().max())


def adam64(p, g, m, v, step, lr, b1, b2, eps, wd):
    p, g, m, v = p.double(), g.double(), m.double(), v.double()
    g = g + wd * p
    m = m + (1 - b1) * (g - m)
    v = v * b2 + (1 - b2) * g * g
    step_size = lr / (1 - b1 ** step)
    denom = v.sqrt() / math.sqrt(1 - b2 ** step) + eps
    return p - step_size * m / denom, m, v


def warm_state(params, gen, step=7):
    """A state_dict for `params` at `step` with random moments, loadable by both optimisers."""
    state = {i: {"step": torch.tensor(float(step)), "exp_avg": (torch.randn(p.shape, generator=gen) * 1e-2).to(DEV),
                 "exp_avg_sq": (torch.rand(p.shape, generator=gen) * 1e-4).to(DEV)} for i, p in enumerate(params)}
    return state


@pytest.mark.parametrize("wd", [0.0, 1e-4])
@pytest.mark.parametrize("name", list(PARAM_SETS))
def test_one_step_against_float64(name, wd):
    base = params_of(name)
    gen = torch.Generator().manual_seed(1)
    ours, theirs, oa, ta = make_pair(base, lr=1e-3, weight_decay=wd)
    sd = ta.state_dict()
    sd["state"] = warm_state(base, gen)
    oa.load_state_dict(copy.deepcopy(sd))
    ta.load_state_dict(copy.deepcopy(sd))
    grads = synth_grads(base, gen)
    for p, q, g in zip(ours, theirs, grads):
        p.grad, q.grad = g.clone(), g.clone()
    oa.step()
    ta.step()
    worst_ulps = 0
    for i, (p, q, p0, g) in enumerate(zip(ours, theirs, base, grads)):
        s = sd["state"][i]
        want = adam64(p0, g, s["exp_avg"], s["exp_avg_sq"], 8, 1e-3, 0.9, 0.999, 1e-8, wd)
        for got, ref, w, what in ((p, q, want[0], "param"), (oa.state[p]["exp_avg"], ta.state[q]["exp_avg"], want[1],
                                                               "exp_avg"),
                                  (oa.state[p]["exp_avg_sq"], ta.state[q]["exp_avg_sq"], want[2], "exp_avg_sq")):
            e_ours = float((got.detach().double() - w).abs().max())
            e_torch = float((ref.detach().double() - w).abs().max())
            one_ulp = float(w.abs().max()) * 2.0 ** -23
            assert e_ours <= ADAM_ERR_FACTOR * e_torch + one_ulp, (name, i, what, e_ours, e_torch)
            worst_ulps = max(worst_ulps, ulps(got.detach(), ref.detach()))
        assert oa.state[p]["step"].item() == ta.state[q]["step"].item() == 8.0
    print(f"{name} wd={wd}: largest distance from torch.optim.Adam (foreach) {worst_ulps} ulp")


@pytest.mark.parametrize("name", list(PARAM_SETS))
def test_hundred_steps_follow_torch(name):
    base = params_of(name, seed=2)
    ours, theirs, oa, ta = make_pair(base, lr=1e-3, weight_decay=1e-4)
    gen = torch.Generator().manual_seed(3)
    for _ in range(100):
        for p, q, g in zip(ours, theirs, synth_grads(base, gen)):
            p.grad, q.grad = g + 1e-2 * p.detach(), g + 1e-2 * q.detach()
        oa.step()
        ta.step()
    for i, (p, q) in enumerate(zip(ours, theirs)):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-5, atol=2e-6, msg=f"{name} param {i}")
        for k in ("exp_avg", "exp_avg_sq"):
            torch.testing.assert_close(oa.state[p][k], ta.state[q][k], rtol=1e-4, atol=1e-9, msg=f"{name} {k} {i}")


def odd_views(shapes, gen):
    """Parameters that are views into one buffer at element offsets 1, 2, 3 (storage offsets not 16-byte aligned)."""
    buf = torch.randn(sum(math.prod(s) for s in shapes) + 4 * len(shapes), generator=gen).to(DEV)
    out, off = [], 1
    for s in shapes:
        n = math.prod(s)
        out.append(buf[off:off + n].view(s))
        off += n + 1 + off % 3
    return out


def test_edge_cases():
    """1-element tensors, unaligned storage offsets, a parameter whose grad is None on some steps (its step count falls
    behind), more tensors than one launch's table holds (Adam: 3 launches, clip: 4)."""
    gen = torch.Generator().manual_seed(4)
    shapes = [(1,), (1, 1), (3,), (5, 7), (129,)] + [(1 + (k * 37) % 50,) for k in range(1100)]
    values = odd_views(shapes, gen)
    ours = [torch.nn.Parameter(v) for v in odd_views(shapes, gen)]
    with torch.no_grad():
        for p, v in zip(ours, values):
            p.copy_(v)
            p.grad = None
    theirs = [torch.nn.Parameter(p.detach().clone()) for p in ours]
    assert sum(p.data_ptr() % 16 != 0 for p in ours) > len(ours) // 2
    oa, ta = Adam(ours, lr=1e-2, weight_decay=1e-4), torch.optim.Adam(theirs, lr=1e-2, weight_decay=1e-4)
    gsrc, gbuf = odd_views(shapes, gen), odd_views(shapes, gen)
    table_splits = 0
    for step in range(6):
        for i, (p, q, g, gv) in enumerate(zip(ours, theirs, gsrc, gbuf)):
            skip = i % 5 == 2 and step % 2 == 0
            if not skip:
                gv.copy_(g * (step + 1))                          # unaligned gradient views for ours
            p.grad = None if skip else gv
            q.grad = None if skip else g * (step + 1)
        n0 = _native.launch_count()
        norm = clip_grad_norm_(ours, 0.5)
        oa.step()
        launches = _native.launch_count() - n0
        ref_norm = torch.nn.utils.clip_grad_norm_(theirs, 0.5)
        ta.step()
        torch.testing.assert_close(norm, ref_norm, rtol=1e-6, atol=0)
        live = sum(p.grad is not None for p in ours)
        assert launches == 2 * -(-live // 1024) + -(-live // 512)
        table_splits += launches == 7
    assert table_splits == 3
    for i, (p, q) in enumerate(zip(ours, theirs)):
        assert oa.state[p]["step"].item() == ta.state[q]["step"].item()
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-5, atol=1e-6, msg=f"tensor {i}")
    assert oa.state[ours[3]]["step"].item() == 6.0 and oa.state[ours[7]]["step"].item() == 3.0


def test_adam_refuses_on_the_device():
    with pytest.raises(NotImplementedError, match="not contiguous"):
        Adam([torch.nn.Parameter(torch.zeros(4, 3, device=DEV).t())])
    with pytest.raises(NotImplementedError, match="cpu"):
        Adam([torch.nn.Parameter(torch.zeros(3, device=DEV)), torch.nn.Parameter(torch.zeros(3))])
    p = torch.nn.Parameter(torch.zeros(4, 3, device=DEV))
    opt = Adam([p])
    p.grad = torch.zeros(3, 4, device=DEV).t()
    with pytest.raises(NotImplementedError, match="not contiguous"):
        opt.step()


def test_state_dict_round_trip_with_torch():
    base = params_of("mdtc_small")
    ours, theirs, oa, ta = make_pair(base, lr=1e-3, weight_decay=1e-4)
    gen = torch.Generator().manual_seed(5)
    for _ in range(3):
        for p, q, g in zip(ours, theirs, synth_grads(base, gen)):
            p.grad, q.grad = g.clone(), g.clone()
        oa.step()
        ta.step()
    s_ours, s_torch = oa.state_dict(), ta.state_dict()
    strip = lambda groups: [{k: v for k, v in g.items() if k != "foreach"} for g in groups]
    assert strip(s_ours["param_groups"]) == strip(s_torch["param_groups"])
    assert s_ours["state"].keys() == s_torch["state"].keys()
    for k, st in s_ours["state"].items():
        assert list(st) == ["step", "exp_avg", "exp_avg_sq"]
        assert st["step"].device.type == "cpu" and st["step"].dtype == torch.float32 and st["step"].dim() == 0
        assert st["exp_avg"].shape == base[k].shape and st["exp_avg"].device == DEV
    # resume each run on the other optimiser: both continue the same trajectory
    ours2, theirs2 = [torch.nn.Parameter(p.detach().clone()) for p in theirs], \
        [torch.nn.Parameter(p.detach().clone()) for p in ours]
    oa2, ta2 = Adam(ours2, lr=1e-3), torch.optim.Adam(theirs2, lr=1e-3)
    oa2.load_state_dict(copy.deepcopy(s_torch))
    ta2.load_state_dict(copy.deepcopy(s_ours))
    for _ in range(3):
        grads = synth_grads(base, gen)
        for pairs in ((ours, ours2), (theirs, theirs2)):
            for p, q, g in zip(*pairs, grads):
                p.grad, q.grad = g.clone(), g.clone()
        for o in (oa, ta, oa2, ta2):
            o.step()
    for a, b, c, d in zip(ours, theirs, ours2, theirs2):
        torch.testing.assert_close(c.detach(), b.detach(), rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(d.detach(), a.detach(), rtol=1e-5, atol=1e-6)


def test_lr_is_read_every_step():
    base = params_of("tcn")
    ours, theirs, oa, ta = make_pair(base, lr=1e-3)
    so = torch.optim.lr_scheduler.ReduceLROnPlateau(oa, factor=0.5, patience=0)
    st = torch.optim.lr_scheduler.ReduceLROnPlateau(ta, factor=0.5, patience=0)
    gen = torch.Generator().manual_seed(6)
    for k in range(4):
        for p, q, g in zip(ours, theirs, synth_grads(base, gen)):
            p.grad, q.grad = g.clone(), g.clone()
        oa.step()
        ta.step()
        so.step(1.0)
        st.step(1.0)
    assert oa.param_groups[0]["lr"] == ta.param_groups[0]["lr"] < 1e-3
    for p, q in zip(ours, theirs):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-5, atol=1e-6)


def test_param_groups():
    base = params_of("gru")
    a = [torch.nn.Parameter(t.clone()) for t in base]
    b = [torch.nn.Parameter(t.clone()) for t in base]
    groups = lambda ps: [dict(params=ps[:5], lr=1e-2, betas=(0.8, 0.99)), dict(params=ps[5:], weight_decay=1e-3)]
    oa, ta = Adam(groups(a), lr=1e-3), torch.optim.Adam(groups(b), lr=1e-3)
    gen = torch.Generator().manual_seed(7)
    for _ in range(5):
        for p, q, g in zip(a, b, synth_grads(base, gen)):
            p.grad, q.grad = g.clone(), g.clone()
        oa.step()
        ta.step()
    for p, q in zip(a, b):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-5, atol=1e-6)


def clip_pair(name, gen, scale=1.0):
    base = params_of(name)
    grads = synth_grads(base, gen, scale)
    ours = [torch.nn.Parameter(t.clone()) for t in base]
    theirs = [torch.nn.Parameter(t.clone()) for t in base]
    for p, q, g in zip(ours, theirs, grads):
        p.grad, q.grad = g.clone(), g.clone()
    return ours, theirs, grads


@pytest.mark.parametrize("name", list(PARAM_SETS))
def test_clip_against_torch_and_float64(name):
    gen = torch.Generator().manual_seed(8)
    ours, theirs, grads = clip_pair(name, gen)
    for max_norm in (0.5, 1e6):                  # clipped, and coef 1 (every gradient still multiplied by 1)
        for p, q, g in zip(ours, theirs, grads):
            p.grad.copy_(g)
            q.grad.copy_(g)
        norm = clip_grad_norm_(ours, max_norm)
        ref = torch.nn.utils.clip_grad_norm_(theirs, max_norm)
        assert norm.shape == () and norm.dtype == torch.float32 and norm.device == DEV
        n64 = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads))
        assert abs(float(norm) - float(ref)) <= 1e-6 * float(ref)
        assert abs(float(norm) - n64) <= abs(float(ref) - n64)
        coef = torch.clamp(max_norm / (norm + 1e-6), max=1.0)
        for p, g in zip(ours, grads):
            assert torch.equal(p.grad, g * coef)


@pytest.mark.parametrize("bad", [math.inf, -math.inf, math.nan])
def test_clip_non_finite_as_torch(bad):
    gen = torch.Generator().manual_seed(9)
    ours, theirs, grads = clip_pair("tcn", gen)
    for ps in (ours, theirs):
        ps[3].grad.view(-1)[5] = bad
    norm = clip_grad_norm_(ours, 5.0)
    ref = torch.nn.utils.clip_grad_norm_(theirs, 5.0)
    assert (math.isnan(float(norm)) and math.isnan(float(ref))) or float(norm) == float(ref)
    for p, q in zip(ours, theirs):
        torch.testing.assert_close(p.grad, q.grad, rtol=0, atol=0, equal_nan=True)
    # error_if_nonfinite: torch's error, gradients untouched
    ours, theirs, grads = clip_pair("tcn", gen)
    for ps in (ours, theirs):
        ps[3].grad.view(-1)[5] = bad
    before = [p.grad.clone() for p in ours]
    with pytest.raises(RuntimeError) as theirs_err:
        torch.nn.utils.clip_grad_norm_(theirs, 5.0, error_if_nonfinite=True)
    with pytest.raises(RuntimeError) as ours_err:
        clip_grad_norm_(ours, 5.0, error_if_nonfinite=True)
    assert str(ours_err.value) == str(theirs_err.value)
    for p, b in zip(ours, before):
        torch.testing.assert_close(p.grad, b, rtol=0, atol=0, equal_nan=True)


def test_clip_error_if_nonfinite_on_finite_grads():
    gen = torch.Generator().manual_seed(10)
    a, _, grads = clip_pair("gru", gen)
    b = [torch.nn.Parameter(p.detach().clone()) for p in a]
    for p, g in zip(b, grads):
        p.grad = g.clone()
    n0 = _native.launch_count()
    na = clip_grad_norm_(a, 0.1, error_if_nonfinite=True)
    assert _native.launch_count() - n0 == 4
    nb = clip_grad_norm_(b, 0.1)
    assert torch.equal(na, nb) and all(torch.equal(p.grad, q.grad) for p, q in zip(a, b))


def test_determinism_and_launch_counts():
    base = params_of("mdtc")
    gen = torch.Generator().manual_seed(11)
    grads = synth_grads(base, gen)
    runs = []
    for _ in range(2):
        ps = [torch.nn.Parameter(t.clone()) for t in base]
        for p, g in zip(ps, grads):
            p.grad = g.clone()
        opt = Adam(ps, lr=1e-3, weight_decay=1e-4)
        counts = []
        for _ in range(2):
            n0 = _native.launch_count()
            norm = clip_grad_norm_(ps, 0.05)
            counts.append(_native.launch_count() - n0)
            n0 = _native.launch_count()
            opt.step()
            counts.append(_native.launch_count() - n0)
        assert counts == [2, 1, 2, 1]
        runs.append([norm] + [p.detach() for p in ps] + [p.grad for p in ps]
                    + [opt.state[p][k] for p in ps for k in ("exp_avg", "exp_avg_sq")])
    assert all(torch.equal(x, y) for x, y in zip(*runs))


def test_step_moves_version_counters():
    """The kernels write through raw pointers; the version counters still move: a KWSModel's eval repacks the new
    weights, and autograd notices a step between a forward and its backward."""
    cfg = model_config("mdtc_small")
    model = synth.randomize_(init_model(cfg), seed=12).to(DEV)
    feats = torch.randn(2, 30, 80, generator=torch.Generator().manual_seed(13)).to(DEV)
    with torch.no_grad():
        y_before, _ = model.eval()(feats)                       # packs the eval kernel's weights
    model.enable_training().train()
    y, _ = model(feats)
    y.sum().backward()
    opt = Adam(model.parameters(), lr=1e-2)
    clip_grad_norm_(model.parameters(), 1.0)
    opt.step()
    fresh = init_model(cfg)
    fresh.load_state_dict({k: v.cpu() for k, v in model.state_dict().items()})
    with torch.no_grad():
        y_after, _ = model.eval()(feats)
        y_fresh, _ = fresh.to(DEV).eval()(feats)
    assert not torch.equal(y_after, y_before)
    assert torch.equal(y_after, y_fresh)

    w = torch.nn.Parameter(torch.randn(8, device=DEV))
    loss = (w * w).sum()                                        # saves w for the backward
    w.grad = torch.ones_like(w)
    Adam([w]).step()
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        loss.backward()


def executor_train(model, opt, clip_fn, batches, crit_name, seed):
    """Executor.train (executor.py:28-68): loss -> backward -> clip -> isfinite -> step.  [(loss, stepped)]."""
    model.train()
    torch.manual_seed(seed)
    log = []
    for b in batches:
        target = b["target"][:, 0] if b["target"].shape[1] == 1 else b["target"]
        logits, _ = model(b["feats"].to(DEV))
        loss, _ = criterion(crit_name, logits, target.to(DEV), b["feats_lengths"].to(DEV),
                            target_lengths=b["target_lengths"].to(DEV), min_duration=0, validation=False)
        opt.zero_grad()
        loss.backward()
        grad_norm = clip_fn(model.parameters(), 5.0)
        stepped = bool(torch.isfinite(grad_norm))
        if stepped:
            opt.step()
        log.append((loss.item(), stepped))
    return log


def executor_case(case):
    gen = torch.Generator().manual_seed(14)
    if case == "mdtc_max_pooling":
        model = synth.randomize_(init_model(model_config("mdtc_small")), seed=15).to(DEV).enable_training()
        batches = []
        for _ in range(5):
            lens = torch.randint(30, 61, (8,), generator=gen)
            lens[0] = 60
            batches.append(dict(feats=torch.randn(8, 60, 80, generator=gen), target=torch.tensor([[0]] * 8),
                                feats_lengths=lens, target_lengths=torch.ones(8, dtype=torch.long)))
        return model, batches, "max_pooling"
    if case == "mdtc_head_ce":
        torch.manual_seed(16)
        model = synth.randomize_(init_model(head_config("mdtc_global")), seed=16).to(DEV)
        model.enable_training(device_dropout=True)
        batches = [dict(feats=torch.randn(16, 98, 80, generator=gen), target=torch.randint(0, 11, (16, 1), generator=gen),
                        feats_lengths=torch.full((16,), 98), target_lengths=torch.ones(16, dtype=torch.long))
                   for _ in range(5)]
        return model, batches, "ce"
    model = synth.randomize_(init_model(model_config("fsmn", input_dim=400, output_dim=2599, activation="identity")),
                             seed=17).to(DEV)
    batches = []
    for _ in range(5):
        lens = torch.randint(12, 31, (4,), generator=gen)
        lens[0] = 30
        batches.append(dict(feats=torch.randn(4, 30, 400, generator=gen), target=torch.randint(1, 2599, (4, 3), generator=gen),
                            feats_lengths=lens, target_lengths=torch.randint(1, 4, (4,), generator=gen)))
    return model, batches, "ctc"


@pytest.mark.parametrize("case", ["mdtc_max_pooling", "mdtc_head_ce", "fsmn_ctc"])
def test_executor_train_end_to_end(case):
    model, batches, crit = executor_case(case)
    twin = copy.deepcopy(model)
    logs = [executor_train(model, Adam(model.parameters(), lr=1e-3), clip_grad_norm_, batches, crit, 18),
            executor_train(twin, torch.optim.Adam(twin.parameters(), lr=1e-3), torch.nn.utils.clip_grad_norm_,
                           batches, crit, 18)]
    assert [s for _, s in logs[0]] == [s for _, s in logs[1]]
    # the losses follow; the weights are not compared, since Adam moves a weight whose gradient is zero up to round-off
    # (a conv bias in front of a BatchNorm) by +-lr whatever the sign of that round-off
    for (a, _), (b, _) in zip(*logs):
        assert (math.isinf(a) and math.isinf(b)) or abs(a - b) <= 1e-3 * abs(b), (a, b)
