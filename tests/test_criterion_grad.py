"""GPU tests of the training-criterion gradients (csrc/criterion.cu: max_pool_grad_kernel, ce_grad_kernel,
ctc_beta_kernel, ctc_grad_kernel) against the reference's own loss.py under autograd
(tests/golden/criterion_grad.npz) and the CPU oracle (oracle/kws_criterion_grad_oracle.py).

Tolerances.  max_pooling: the non-zero pattern is exact and the values are within 4 ulp (a handful of float32
divisions, rounded in a different order).  ce and ctc: the error against the float64 gradient is at most GRAD_MULT
times the largest error of the reference's own float32 gradient against float64 over the fixture (or over the random
batch itself), plus an absolute floor of ABS_FLOOR for elements whose float32 reference happens to be exact.  Zero
rows are exactly zero and NaN rows are exactly the reference's."""
import numpy as np
import pytest
import torch

from oracle import kws_criterion_grad_oracle as KG
from oracle import kws_criterion_oracle as K
from tests.test_criterion import peaky_ctc_batch
from tests.test_criterion_grad_host import G, NAMES, grad_inputs
from wekws_b200 import _native, criterion
from wekws_b200.criterion import cross_entropy, ctc_loss, max_pooling_loss

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GRAD_MULT = 8.0
ABS_FLOOR = 2.0 ** -24


def dev(*ts):
    return [None if t is None else t.to(DEV) for t in ts]


def device_grad(ctype, x, t, l, tl, md=0, up=1.0):
    """(loss, gradient) of the device criterion, the loss scaled by `up` before backward()."""
    xd = x.to(DEV).requires_grad_(True)
    t, l, tl = dev(t, l, tl)
    loss, _ = criterion(ctype, xd, t, l, tl, md)
    (loss * up if up != 1.0 else loss).backward()
    return loss.detach(), xd.grad


def spread(names):
    """Largest |float32 - float64| of the reference's finite gradients over the named fixture calls."""
    e = 0.0
    for n in names:
        a, b = G[f"{n}__grad"].astype(np.float64), G[f"{n}__grad64"]
        ok = np.isfinite(b)
        e = max(e, float(np.abs(a - b)[ok].max()))
    return e


def ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize("name", NAMES)
def test_golden_gradients(name):
    ctype, x, t, l, tl, md, up = grad_inputs(name)
    loss, grad = device_grad(ctype, x, t, l, tl, md, up)
    assert grad.dtype == torch.float32 and grad.shape == x.shape and grad.is_cuda
    with torch.no_grad():
        plain, _ = criterion(ctype, *dev(x, t, l, tl), md)
    assert loss.view(torch.int32).item() == plain.view(torch.int32).item()    # the grad path's loss, bit for bit
    got, want, want64 = grad.cpu().numpy(), G[f"{name}__grad"], G[f"{name}__grad64"]
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got == 0, want == 0)
    if ctype == "max_pooling":
        assert int(ulps(got, want).max()) <= 4
        return
    tol = GRAD_MULT * spread([n for n in NAMES if G[f"{n}__type"] == ctype]) + ABS_FLOOR
    ok = np.isfinite(want64)
    assert float(np.abs(got.astype(np.float64) - want64)[ok].max()) <= tol


def saturated_posteriors(B, T, D, gen):
    """Posteriors as late in training: many exactly 1.0 (ties at the top) and many below the clamp (0, 1e-9)."""
    x = torch.rand(B, T, D, generator=gen) ** 3
    r = torch.rand(B, T, D, generator=gen)
    x[r < 0.10] = 1.0
    x[(r >= 0.10) & (r < 0.20)] = 0.0
    x[(r >= 0.20) & (r < 0.25)] = 1e-9
    return x


def test_random_max_pooling_against_oracle():
    gen = torch.Generator().manual_seed(21)
    for B, T, D in ((256, 300, 2), (37, 1000, 5)):
        x = saturated_posteriors(B, T, D, gen)
        x[1] = 0.0                                           # every frame ties, all outside the clamp for a keyword
        t = torch.randint(-1, D + 1, (B,), generator=gen)
        lens = torch.randint(1, T + 1, (B,), generator=gen)
        lens[3] = T
        for md in (0, 7):
            _, grad = device_grad("max_pooling", x, t, lens, None, md)
            _, ref = KG.criterion_grad("max_pooling", x, t, lens, None, md)
            got, want = grad.cpu().numpy(), ref.numpy()
            assert np.array_equal(got == 0, want == 0) and int(ulps(got, want).max()) <= 4
            assert (np.count_nonzero(want, axis=1) > 1).any()        # ties were split


def test_random_ce_against_oracle():
    gen = torch.Generator().manual_seed(22)
    x = torch.randn(4096, 11, generator=gen) * 4
    t = torch.randint(0, 11, (4096,), generator=gen)
    t[::17] = -100
    _, grad = device_grad("ce", x, t, None, None)
    _, ref32 = KG.criterion_grad("ce", x, t, None)
    _, ref64 = KG.criterion_grad("ce", x, t, None, dtype=torch.float64)
    got = grad.cpu()
    assert not got[t == -100].any() and got[t != -100].all()
    tol = GRAD_MULT * float((ref32.double() - ref64).abs().max()) + ABS_FLOOR
    assert float((got.double() - ref64).abs().max()) <= tol


def test_random_recipe_size_ctc_against_oracle():
    """B = 256, T <= 1000, V = 2599, labels up to 200 tokens with repeats.  A subset of utterances is compared with
    the oracle on the CPU (a batch of its own: utterances are independent up to the 1 / B factor); every row's
    gradient sums to ~0 and the occupancy part of every feasible frame sums to 1.  The backward allocates nothing of
    B*T*V elements but the gradient it returns."""
    B, T, V, L = 256, 1000, 2599, 200
    x, tgt, lens, tl = peaky_ctc_batch(B, T, V, L, seed=11)
    tgt[0, 1::7] = tgt[0, 0]                                 # the 200-token label repeats a token, apart ...
    tgt[0, 50:53] = tgt[0, 49]                               # ... and adjacent
    lens[5], tl[5] = 20, 30                                  # infeasible
    tgt[5, :30] = torch.arange(1, 31)
    lens[6], tl[6] = 0, 0                                    # no frames, empty label
    xd = x.to(DEV).requires_grad_(True)
    tgt_d, lens_d, tl_d = dev(tgt, lens, tl)
    loss, _, out = ctc_loss(xd, tgt_d, lens_d, tl_d, terms=True)
    assert not out["term"].requires_grad
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()
    (grad,) = torch.autograd.grad(loss, xd, retain_graph=True)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - before
    assert extra < 1.01 * x.numel() * 4, extra              # the gradient itself and nothing else of its size
    (again,) = torch.autograd.grad(loss, xd)                 # reuses the occupancies the first call formed
    assert torch.equal(grad.view(torch.int32), again.view(torch.int32))

    valid = (torch.arange(T)[None, :] < lens[:, None]).to(DEV)
    feasible = torch.isfinite(out["term"])
    assert feasible.sum() == B - 1 and not feasible[5]
    assert torch.isnan(grad[5, :20]).all() and not grad[5, 20:].any()
    assert not grad[~valid].any()
    rows = grad[valid & feasible[:, None]]
    assert torch.isfinite(rows).all()
    # softmax sums to 1 and so does the occupancy, the exp of float32 log-sums as large as the utterance's loss
    # (thousands here, accumulated over up to 1000 frames): within 3 % per frame, i.e. 0.03 / B on the row's sum
    assert float(rows.sum(1).abs().max()) < 0.03 / B
    del rows, again

    sub = [0, 1, 2, 6, 17, 255]
    xs = x[sub]
    _, ref32 = KG.criterion_grad("ctc", xs, tgt[sub], lens[sub], tl[sub])
    _, ref64 = KG.criterion_grad("ctc", xs, tgt[sub], lens[sub], tl[sub], dtype=torch.float64)
    got = grad[sub].cpu().double() * (B / len(sub))          # 1 / B of the whole batch -> 1 / len(sub)
    tol = GRAD_MULT * float((ref32.double() - ref64).abs().max()) + ABS_FLOOR
    assert float((got - ref64).abs().max()) <= tol, (float((got - ref64).abs().max()), tol)
    # occupancy per frame: softmax - B * gradient, summed over the vocabulary, is 1 on the frames of utterance 0
    occ = xs[0].double().softmax(1) - got[0] * len(sub)
    assert float((occ.sum(1)[:int(lens[0])] - 1).abs().max()) < 0.03


@pytest.mark.parametrize("name", ["mp_rand", "ce0", "ctc0"])
def test_upstream_scale_and_determinism(name):
    ctype, x, t, l, tl, md, _ = grad_inputs(name)
    _, g1 = device_grad(ctype, x, t, l, tl, md)
    _, g1b = device_grad(ctype, x, t, l, tl, md)
    assert torch.equal(g1.view(torch.int32), g1b.view(torch.int32))
    _, g3 = device_grad(ctype, x, t, l, tl, md, up=3.0)
    assert torch.equal(g3, g1 * 3.0)                         # upstream * (unit gradient), one float32 multiplication


class Head(torch.nn.Module):
    """A small stand-in for the reference's models: returns (logits, cache) like them."""

    def __init__(self, idim, odim, sigmoid):
        super().__init__()
        self.net = torch.nn.Sequential(torch.nn.Linear(idim, 16), torch.nn.Tanh(), torch.nn.Linear(16, odim),
                                       torch.nn.Sigmoid() if sigmoid else torch.nn.Identity())

    def forward(self, feats):
        return self.net(feats), None


def oracle_criterion(type, logits, target, lengths, target_lengths=None, min_duration=0, validation=False):
    if type == "max_pooling":
        return KG.max_pooling_loss_graph(logits, target, lengths, min_duration), 0.0
    return K.criterion(type, logits, target, lengths, target_lengths, min_duration, validation)


def train_batches(ctype, gen, n=5):
    out = []
    for k in range(n):
        if ctype == "ce":
            b = dict(feats=torch.randn(24, 10, generator=gen), target=torch.randint(0, 4, (24, 1), generator=gen),
                     feats_lengths=torch.ones(24, dtype=torch.int64), target_lengths=torch.ones(24, dtype=torch.int64))
        elif ctype == "max_pooling":
            lens = torch.randint(5, 31, (12,), generator=gen)
            lens[0] = 30
            b = dict(feats=torch.randn(12, 30, 10, generator=gen), target=torch.randint(-1, 2, (12, 1), generator=gen),
                     feats_lengths=lens, target_lengths=torch.ones(12, dtype=torch.int64))
        else:
            lens = torch.randint(12, 31, (8,), generator=gen)
            tl = torch.randint(1, 5, (8,), generator=gen)
            if k == 2:
                lens[3], tl[3] = 2, 4                        # infeasible: this batch's step is skipped
            b = dict(feats=torch.randn(8, 30, 10, generator=gen), target=torch.randint(1, 6, (8, 4), generator=gen),
                     feats_lengths=lens, target_lengths=tl)
        out.append(b)
    return out


@pytest.mark.parametrize("ctype", ["max_pooling", "ce", "ctc"])
def test_training_through_a_model(ctype):
    """Executor.train's pattern -- model(feats), criterion, loss.backward(), clip_grad_norm_, optimizer.step() -- with
    the device criterion under a torch model on the device, against the same model on the CPU with the oracle
    criterion: first the parameter gradients of one batch, then five Adam steps."""
    gen = torch.Generator().manual_seed(31)
    odim = {"max_pooling": 2, "ce": 4, "ctc": 6}[ctype]
    torch.manual_seed(5)
    cpu = Head(10, odim, ctype == "max_pooling")
    gpu = Head(10, odim, ctype == "max_pooling")
    gpu.load_state_dict(cpu.state_dict())
    gpu.to(DEV)
    args = {"criterion": ctype, "grad_clip": 5.0, "min_duration": 2}
    batches = train_batches(ctype, gen)

    for model, crit, device in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV)):
        KG.train(crit, model, torch.optim.SGD(model.parameters(), lr=0.0), batches[:1], torch.device(device), args)
    for (n, p), q in zip(cpu.named_parameters(), gpu.parameters()):
        assert torch.allclose(q.grad.cpu(), p.grad, rtol=1e-4, atol=1e-6), n

    logs = [KG.train(crit, model, torch.optim.Adam(model.parameters(), lr=1e-2), batches, torch.device(device), args)
            for model, crit, device in ((cpu, oracle_criterion, "cpu"), (gpu, criterion, DEV))]
    assert [s for _, s in logs[0]] == [s for _, s in logs[1]] == [ctype != "ctc" or k != 2 for k in range(5)]
    for (a, _), (b, _) in zip(*logs):
        assert (np.isinf(a) and np.isinf(b)) or abs(a - b) <= 1e-3 * abs(a)       # five steps of float32 drift


def test_launch_counts():
    x = torch.rand(4, 10, 2, device=DEV)
    lens = torch.full((4,), 10, device=DEV)
    t = torch.tensor([0, 1, -1, 0], device=DEV)
    lc = torch.randn(4, 40, 8, device=DEV)
    lab = torch.tensor([[1, 2], [3, 3], [4, -1], [5, 6]], device=DEV)
    tl = torch.tensor([2, 2, 1, 2], device=DEV)
    calls = ((lambda v: criterion("max_pooling", v, t, lens), x, 2, 1),
             (lambda v: criterion("ce", v, t.clamp(min=0), None), x[:, 0].contiguous(), 2, 1),
             (lambda v: criterion("ctc", v, lab, lens * 4, tl), lc, 3, 2),
             (lambda v: criterion("ctc", v, lab, lens * 4, tl, validation=True), lc, 5, 2))
    for call, inp, fwd, bwd in calls:
        n0 = _native.launch_count()
        call(inp)                                            # the forward-only path: unchanged
        with torch.no_grad():
            call(inp.clone().requires_grad_(True))
        assert _native.launch_count() - n0 == 2 * fwd
        v = inp.clone().requires_grad_(True)
        n0 = _native.launch_count()
        loss, _ = call(v)
        assert _native.launch_count() - n0 == fwd
        loss.backward(retain_graph=True)
        assert _native.launch_count() - n0 == fwd + bwd
        first = v.grad.clone()
        v.grad = None
        loss.backward()                                      # a second backward of a ctc loss reuses the occupancies
        assert _native.launch_count() - n0 == fwd + bwd + 1
        assert torch.equal(v.grad.view(torch.int32), first.view(torch.int32))


def test_direct_entry_points_and_refusals():
    x = torch.rand(4, 10, 2, device=DEV, requires_grad=True)
    lens = torch.full((4,), 10, device=DEV)
    t = torch.tensor([0, 1, -1, 0], device=DEV)
    loss, _, out = max_pooling_loss(x, t, lens, terms=True)
    assert loss.requires_grad and not out["term"].requires_grad
    (g,) = torch.autograd.grad(loss, x, create_graph=True)
    assert not g.requires_grad                               # once_differentiable: the gradient is a constant,
    with pytest.raises(RuntimeError):                        # so differentiating it again is refused
        g.sum().backward()
    loss, _, out = cross_entropy(x[:, 0], t.clamp(min=0), terms=True)
    assert loss.requires_grad and not out["term"].requires_grad
    loss.backward()                                          # through the slice: the gradient lands in x
    assert x.grad.shape == x.shape and not x.grad[:, 1:].any() and x.grad[:, 0].any()
    loss, _ = criterion("max_pooling", x, t, lens)
    with pytest.raises(RuntimeError):                        # autograd refuses a gradient that is not the loss' shape
        loss.backward(torch.ones(2, device=DEV))
    with torch.no_grad():
        loss, _ = criterion("max_pooling", x, t, lens)
    assert not loss.requires_grad
