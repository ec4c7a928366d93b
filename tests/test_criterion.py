"""GPU tests of wekws_b200.criterion (csrc/criterion.cu) against the reference's own criterion() / Executor.cv
(tests/golden/criterion.npz) and the CPU restatement (oracle/kws_criterion_oracle.py).

Tolerances.  max_pooling folds its terms in the reference's order, so its loss is within 4 ulp of the reference's
float32 value (the terms differ by logf ulps only).  ce and ctc go through torch's own reductions, whose order is not
reproducible; their bound is LOSS_SPREAD_MULT times the largest relative gap between the reference's float32 loss and
the same loss in float64 over the fixtures (or over the random batch itself), i.e. a small multiple of the
reference's own float32 error.  Accuracies, decoded hypotheses and inf are exact."""
import math

import numpy as np
import pytest
import torch

from oracle import kws_criterion_oracle as K
from oracle import kws_oracle as O
from tests.conftest import golden
from tests.head_cases import build_head_model
from tests.test_criterion_host import Echo, call_inputs, cv_batches
from tests.test_stream_spotter import _model
from wekws_b200 import _native, context_expansion, criterion, init_model, model_config, synth
from wekws_b200.criterion import ctc_loss, max_pooling_loss

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
G = golden("criterion")
NAMES = [str(n) for n in G["names"]]
LOSS_SPREAD_MULT = 8.0


def rel_spread(names):
    """Largest |float32 - float64| / |float64| of the reference's finite losses (batch and per utterance)."""
    r = []
    for n in names:
        if f"{n}__loss64" not in G:
            continue
        pairs = [(np.float64(G[f"{n}__loss"]), G[f"{n}__loss64"])]
        if f"{n}__utt_loss" in G:
            pairs += list(zip(G[f"{n}__utt_loss"].astype(np.float64), G[f"{n}__utt_loss64"]))
        r += [abs(a - b) / abs(b) for a, b in pairs if np.isfinite(b) and b != 0]
    return max(r)


def ulp_diff(a, b):
    ia, ib = np.array([a], np.float32).view(np.int32)[0], np.array([b], np.float32).view(np.int32)[0]
    return abs(int(ia) - int(ib))


def close_or_same(got, want, rel):
    got, want = float(got), float(want)
    if math.isnan(want) or math.isinf(want):
        return (math.isnan(got) and math.isnan(want)) or got == want
    return abs(got - want) <= rel * abs(want)


def to_dev(ctype, x, t, l, tl):
    return (x.to(DEV), t.to(DEV), None if l is None else l.to(DEV), None if tl is None else tl.to(DEV))


@pytest.mark.parametrize("name", NAMES)
def test_golden_calls(name):
    ctype, x, t, l, tl, md, val = call_inputs(name)
    xd, td, ld, tld = to_dev(ctype, x, t, l, tl)
    err = str(G[f"{name}__error"])
    if err:
        with pytest.raises(Exception) as e:
            criterion(ctype, xd, td, ld, tld, md, val)
        assert type(e.value).__name__ == err
        return
    loss, acc = criterion(ctype, xd, td, ld, tld, md, val)
    want = float(G[f"{name}__loss"])
    assert loss.is_cuda and loss.dtype == torch.float32 and loss.dim() == 0 and isinstance(acc, float)
    assert acc == float(G[f"{name}__acc"]), (acc, float(G[f"{name}__acc"]))
    if ctype == "max_pooling":
        assert (math.isnan(want) and math.isnan(float(loss))) or ulp_diff(float(loss), want) <= 4
        return
    rel = LOSS_SPREAD_MULT * rel_spread([n for n in NAMES if G[f"{n}__type"] == ctype])
    assert close_or_same(loss.item(), want, rel), (loss.item(), want, rel)
    if ctype == "ctc":
        _, _, out = ctc_loss(xd, td, ld, tld, val, terms=True)
        for got, w in zip(out["term"].cpu().tolist(), G[f"{name}__utt_loss"].tolist()):
            assert close_or_same(got, w, rel), (got, w)
        if f"{name}__best" in G:
            assert np.array_equal(out["best"].cpu().numpy(), G[f"{name}__best"])
            calc = G[f"{name}__calc"]
            assert out["correct"].cpu().tolist() == (calc[:, 0] - calc[:, 2] - calc[:, 3] - calc[:, 4]).tolist()


@pytest.mark.parametrize("name", [str(n) for n in G["cv_names"]])
def test_executor_cv_totals(name):
    ctype = str(G[f"{name}__type"])
    loss, acc = K.cv(criterion, Echo(), cv_batches(name), torch.device(DEV), {"criterion": ctype})
    assert acc == float(G[f"{name}__acc"])
    rel = 4 * 2.0 ** -23 if ctype == "max_pooling" else LOSS_SPREAD_MULT * rel_spread(
        [n for n in NAMES if G[f"{n}__type"] == ctype])
    assert close_or_same(loss, float(G[f"{name}__loss"]), rel)


def peaky_ctc_batch(B, Tmax, V, Lmax, seed):
    """Recipe-sized logits that spell the first 30 tokens of each label (so no decode outgrows 64 tokens; the loss
    still sees the whole label): every frame's top tokens stand well apart (lifts from a small set over a zero
    background), so the device and CPU softmax decode alike."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(Tmax // 2, Tmax + 1, (B,), generator=g)
    lens[0] = Tmax
    tl = torch.randint(0, Lmax + 1, (B,), generator=g)
    tl[0], tl[1] = Lmax, 0
    tgt = torch.randint(1, V, (B, Lmax), generator=g)
    tgt[torch.arange(Lmax)[None, :] >= tl[:, None]] = -1
    x = torch.zeros(B, Tmax, V)
    for b in range(B):
        n, L = int(lens[b]), int(tl[b])
        lab = tgt[b, :min(L, 30)]
        L = lab.numel()
        # blank frames with each spelled token on one frame, evenly spread, and 1 % noise tokens
        hot = torch.zeros(n, dtype=torch.long)
        if L:
            hot[torch.arange(L) * n // L] = lab
        noise = torch.rand(n, generator=g) < 0.01
        hot[noise] = torch.randint(0, V, (int(noise.sum()),), generator=g)
        x[b, torch.arange(n), hot] = 8.0 + torch.randint(0, 3, (n,), generator=g).float()
        alt = torch.randint(0, V, (n,), generator=g)
        keep = alt != hot
        x[b, torch.arange(n)[keep], alt[keep]] = 6.5
    return x, tgt, lens, tl


def test_random_recipe_size_ctc_against_oracle():
    """B = 256, T <= 1000, V = 2599, labels up to 200 tokens: per-utterance losses within the batch's own float32
    spread, inf exactly where the reference has it, the batch loss, and the accuracy decode of 24 utterances
    exactly."""
    B, T, V, L = 256, 1000, 2599, 200
    x, tgt, lens, tl = peaky_ctc_batch(B, T, V, L, seed=11)
    xd = x.to(DEV)
    loss, acc, out = ctc_loss(xd, tgt.to(DEV), lens.to(DEV), tl.to(DEV), validation=True, terms=True)
    ref32 = K.ctc_utterance_losses(x, tgt, lens, tl).double()
    lp64 = x.double().transpose(0, 1).log_softmax(2)
    ref64 = torch.nn.functional.ctc_loss(lp64, tgt, lens, tl, reduction="none")
    fin = torch.isfinite(ref64) & (ref64 != 0)
    rel = LOSS_SPREAD_MULT * float(((ref32 - ref64).abs() / ref64.abs())[fin].max())
    got = out["term"].cpu().double()
    assert torch.equal(torch.isinf(got), torch.isinf(ref32))
    assert float(((got - ref64).abs() / ref64.abs())[fin].max()) <= rel
    assert close_or_same(loss.item(), float(ref32.sum()) / B, rel)
    sub = list(range(24))
    counts = K.ctc_counts(x[sub], tgt[sub], lens[sub], tl[sub])
    assert out["correct"].cpu()[sub].tolist() == [c for _, c in counts]
    hyps = K.best_hypotheses(x[sub], lens[sub])
    best = out["best"].cpu()
    assert [tuple(best[b, 1:1 + best[b, 0]].tolist()) for b in sub] == hyps
    assert any(len(h) >= 25 for h in hyps)                 # long decodes, not trivial ones
    # determinism: two calls give equal bits
    loss2, acc2, out2 = ctc_loss(xd, tgt.to(DEV), lens.to(DEV), tl.to(DEV), validation=True, terms=True)
    assert torch.equal(loss, loss2) and acc == acc2 and torch.equal(out["term"], out2["term"])


def test_random_max_pooling_and_ce_against_oracle():
    g = torch.Generator().manual_seed(5)
    for B, T, D in ((256, 300, 2), (37, 1000, 5)):
        x = torch.rand(B, T, D, generator=g) ** 3
        t = torch.randint(-1, D + 1, (B,), generator=g)
        lens = torch.randint(1, T + 1, (B,), generator=g)
        lens[3] = T
        for md in (0, 7):
            loss, acc = criterion("max_pooling", x.to(DEV), t.to(DEV), lens.to(DEV), min_duration=md)
            rl, ra = K.max_pooling_loss(x, t, lens, md)
            assert acc == ra and ulp_diff(loss.item(), float(rl)) <= 4
            _, _, out = max_pooling_loss(x.to(DEV), t.to(DEV), lens.to(DEV), md, terms=True)
            terms, correct = K.max_pooling_terms(x, t, lens, md)
            assert torch.equal(out["correct"].cpu(), correct)
            assert torch.allclose(out["term"].cpu(), terms, rtol=4 * 2.0 ** -23, atol=0)
    x = torch.randn(4096, 11, generator=g) * 4
    t = torch.randint(0, 11, (4096,), generator=g)
    t[::17] = -100
    loss, acc = criterion("ce", x.to(DEV), t.to(DEV), None)
    rl, ra = K.cross_entropy(x, t)
    r64 = torch.nn.functional.cross_entropy(x.double(), t)
    assert acc == ra
    assert abs(loss.item() - float(r64)) <= max(LOSS_SPREAD_MULT * abs(float(rl) - float(r64)), 2.0 ** -23 * float(r64))


def test_end_to_end_through_models():
    """Device logits from the models, the device criterion against the oracle criterion on the same logits."""
    torch.manual_seed(0)
    # MDTC keyword model, sigmoid posteriors, max-pooling
    m = synth.randomize_(init_model(model_config("mdtc", output_dim=2)), seed=9).eval().to(DEV)
    feats = synth.features(16, 120, 80, seed=3).to(DEV)
    post, _ = m(feats)
    lens = torch.randint(40, post.shape[1] + 1, (16,))
    lens[0] = post.shape[1]
    tgt = torch.tensor([0, 1, -1, -1] * 4)
    loss, acc = criterion("max_pooling", post, tgt.to(DEV), lens.to(DEV))
    rl, ra = K.max_pooling_loss(post.cpu(), tgt, lens)
    assert acc == ra and ulp_diff(loss.item(), float(rl)) <= 4
    # speech-command MDTC with the global head, cross entropy
    _, head = build_head_model("mdtc_global", init_model)
    head = head.to(DEV)
    logits, _ = head(synth.features(32, 98, 80, seed=4).to(DEV))
    t = torch.randint(0, 11, (32,))
    loss, acc = criterion("ce", logits, t.to(DEV), None)
    rl, ra = K.cross_entropy(logits.cpu(), t)
    assert acc == ra and abs(loss.item() - float(rl)) <= 1e-5 * abs(float(rl))
    # FSMN-CTC (context 2/2, frame skip 3) and DS-TCN-CTC: the decode sees exactly forward_softmax's posteriors
    # (at most 62 rows: no prefix can outgrow 64 tokens whatever the random model emits)
    for name, idim, ctx, frames in (("fsmn", 400, True, 186), ("ds_tcn", 40, False, 62)):
        model = _model(name, idim, 48, seed=5, scale=12.0)
        f = synth.features(12, frames, 80 if ctx else 40, seed=6).to(DEV)
        flen = torch.full((12,), frames, dtype=torch.int32)
        flen[3:] = torch.randint(frames // 3, frames + 1, (9,), dtype=torch.int32)
        if ctx:
            f, flen = context_expansion(f, 2, 2, 3, flen)
        logits, _ = model(f.contiguous())
        probs, _ = model.forward_softmax(f.contiguous())
        lens = flen.cpu().to(torch.int64).clamp(max=logits.shape[1])
        labels = torch.randint(1, 48, (12, 6))
        tl = torch.randint(1, 7, (12,))
        loss, acc, out = ctc_loss(logits, labels.to(DEV), lens.to(DEV), tl.to(DEV), validation=True, terms=True)
        ref = K.ctc_utterance_losses(logits.cpu(), labels, lens, tl)
        assert torch.allclose(out["term"].cpu(), ref, rtol=1e-4, atol=0)
        probs_h = probs.cpu()
        best = out["best"].cpu()
        for b in range(12):
            hyps = O.hyps_of(O.ctc_prefix_beam_search(probs_h[b][:int(lens[b])], None, 3, 5))
            want = list(hyps[0][0]) if hyps else []
            assert best[b, 1:1 + best[b, 0]].tolist() == want, (name, b)
            lab = labels[b, :int(tl[b])].tolist()
            assert int(out["correct"][b]) == len(lab) - K.edit_distance(lab, want)


def test_launch_counts():
    x = torch.rand(4, 10, 2, device=DEV)
    lens = torch.full((4,), 10, device=DEV)
    t = torch.tensor([0, 1, -1, 0], device=DEV)
    lc = torch.randn(4, 40, 8, device=DEV)
    lab = torch.tensor([[1, 2], [3, 3], [4, -1], [5, 6]], device=DEV)
    tl = torch.tensor([2, 2, 1, 2], device=DEV)
    for call, want in ((lambda: criterion("max_pooling", x, t, lens), 2),
                       (lambda: criterion("ce", x[:, 0], t.clamp(min=0), None), 2),
                       (lambda: criterion("ctc", lc, lab, lens * 4, tl), 3),
                       (lambda: criterion("ctc", lc, lab, lens * 4, tl, validation=True), 5)):
        n0 = _native.launch_count()
        call()
        assert _native.launch_count() - n0 == want


def test_refuses_bad_input():
    x = torch.rand(4, 10, 2, device=DEV)
    lens = torch.full((4,), 10, device=DEV)
    t = torch.tensor([0, 1, -1, 0], device=DEV)
    with pytest.raises(ValueError):                      # T != lengths.max()
        criterion("max_pooling", x, t, lens - 1)
    with pytest.raises(ValueError):
        criterion("max_pooling", x.double(), t, lens)
    with pytest.raises(ValueError):
        criterion("max_pooling", x, t.float(), lens)
    with pytest.raises(IndexError):
        criterion("ce", x[:, 0], torch.tensor([0, 1, 2, 0], device=DEV), None)
    lc = torch.randn(4, 40, 8, device=DEV)
    lab = torch.tensor([[1, 2], [3, 3], [4, -1], [5, 6]], device=DEV)
    tl = torch.tensor([2, 2, 1, 2], device=DEV)
    with pytest.raises(ValueError):                      # label outside 0..V-1
        criterion("ctc", lc, lab + 5, lens * 4, tl)
    with pytest.raises(ValueError):                      # lengths > T
        criterion("ctc", lc, lab, lens * 5, tl)
    with pytest.raises(ValueError):                      # target_lengths > Lmax
        criterion("ctc", lc, lab, lens * 4, tl + 1)
    with pytest.raises(ValueError):
        criterion("ctc", lc, torch.ones(4, 600, dtype=torch.long, device=DEV), lens * 4, torch.full((4,), 600,
                                                                                                    device=DEV))
    with pytest.raises(RuntimeError, match="utterance 0"):   # a best hypothesis longer than 64 tokens
        n = 200
        alt = torch.full((1, n, 8), -9.0, device=DEV)
        alt[0, torch.arange(n), (torch.arange(n) % 7) + 1] = 9.0
        criterion("ctc", alt, torch.tensor([[1]], device=DEV), torch.tensor([n], device=DEV),
                  torch.tensor([1], device=DEV), validation=True)
    with pytest.raises(SystemExit):
        criterion("bce", x, t, lens)
