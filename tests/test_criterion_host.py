"""CPU tests of the training-criterion restatement (oracle/kws_criterion_oracle.py): against the reference's own
criterion() / Executor.cv (tests/golden/criterion.npz, and live on fresh seeds when the reference sources are
present), the golden's coverage of every quirk, and the device entry point's refusal of CPU input."""
import numpy as np
import pytest
import torch

from oracle import kws_criterion_oracle as K
from tests.conftest import golden, have_reference

G = golden("criterion")
NAMES = [str(n) for n in G["names"]]
CVS = [str(n) for n in G["cv_names"]]


def call_inputs(name):
    """(type, logits, target, lengths, target_lengths, min_duration, validation) of a golden call."""
    g = lambda k: torch.from_numpy(G[f"{name}__{k}"])
    tl = g("target_lengths") if f"{name}__target_lengths" in G else None
    return (str(G[f"{name}__type"]), g("logits"), g("target"), g("lengths") if f"{name}__lengths" in G else None,
            tl, int(G[f"{name}__min_duration"]), bool(G[f"{name}__validation"]))


def cv_batches(name):
    n = int(G[f"{name}__nbatch"])
    return [{k: torch.from_numpy(G[f"{name}_b{i}__{k}"]) for k in ("feats", "target", "feats_lengths", "target_lengths")}
            for i in range(n)]


class Echo(torch.nn.Module):
    def forward(self, feats):
        return feats, None


def same_float(a, b):
    return (np.isnan(a) and np.isnan(b)) or a == b


@pytest.mark.parametrize("name", NAMES)
def test_oracle_equals_golden(name):
    ctype, x, t, l, tl, md, val = call_inputs(name)
    err = str(G[f"{name}__error"])
    if err:
        with pytest.raises(getattr(__builtins__, err, None) or Exception) as e:
            K.criterion(ctype, x, t, l, tl, md, val)
        assert type(e.value).__name__ == err
        return
    loss, acc = K.criterion(ctype, x, t, l, tl, md, val)
    # every loss is the reference's float32 value bit for bit: the oracle runs the same ops in the same order
    assert loss.dtype == torch.float32 and same_float(float(loss), float(G[f"{name}__loss"]))
    assert acc == float(G[f"{name}__acc"])
    if ctype == "ctc":
        assert torch.equal(K.ctc_utterance_losses(x, t, l, tl), torch.from_numpy(G[f"{name}__utt_loss"]))
    if f"{name}__best" in G:
        best, calc = G[f"{name}__best"], G[f"{name}__calc"]
        hyps = K.best_hypotheses(x, l)
        for b, h in enumerate(hyps):
            assert list(h) == best[b, 1:1 + best[b, 0]].tolist()
        for b, (n, c) in enumerate(K.ctc_counts(x, t, l, tl)):
            # Calculator's all / ins + sub + del are the label length / the edit distance
            assert calc[b, 0] == n and n - (calc[b, 2] + calc[b, 3] + calc[b, 4]) == c


@pytest.mark.parametrize("name", CVS)
def test_oracle_cv_equals_golden(name):
    loss, acc = K.cv(K.criterion, Echo(), cv_batches(name), torch.device("cpu"), {"criterion": str(G[f"{name}__type"])})
    assert loss == float(G[f"{name}__loss"]) and acc == float(G[f"{name}__acc"])


def test_golden_covers_every_quirk():
    mp = [n for n in NAMES if G[f"{n}__type"] == "max_pooling"]
    tg = np.concatenate([G[f"{n}__target"] for n in mp])
    assert (tg == -1).any() and (tg < -1).any() and (tg >= 2).any()                       # fillers, out-of-range ids
    assert any(int(G[f"{n}__min_duration"]) > 0 for n in mp)
    assert all(G[f"{n}__lengths"].max() == G[f"{n}__logits"].shape[1] for n in mp)
    assert any((G[f"{n}__lengths"] < G[f"{n}__logits"].shape[1]).any() for n in mp)     # padding
    assert any(np.isnan(G[f"{n}__logits"]).any() for n in mp) and np.isnan(G["mp1_nan__loss"])
    x, l = G["mp0__logits"], G["mp0__lengths"]                                            # argmax tie over D
    cm = np.where(np.arange(x.shape[1])[None, :, None] < l[:, None, None], x, 0).max(1)
    assert (cm == cm.max(1, keepdims=True)).sum(1).max() >= 2
    assert (G["ce0__target"] == -100).any() and np.isnan(G["ce_all_ignored__loss"])
    assert str(G["ce_bad_target__error"]) == "IndexError"
    ce = G["ce0__logits"]
    assert ((ce == ce.max(1, keepdims=True)).sum(1) >= 2).any()
    ctc = [n for n in NAMES if G[f"{n}__type"] == "ctc"]
    labs = [G[f"{n}__target"] for n in ctc if G[f"{n}__target"].ndim == 2]
    assert any(((a[:, 1:] == a[:, :-1]) & (a[:, 1:] >= 0)).any() for a in labs)         # repeated labels
    assert any((G[f"{n}__target_lengths"] == 0).any() for n in ctc)
    assert np.isinf(G["ctc0__loss"]) and np.isinf(G["ctc0__utt_loss"]).sum() == 1          # infeasible utterance
    assert G["ctc_1d__target"].ndim == 1 and str(G["ctc_1d_val__error"]) == "IndexError"
    assert str(G["ctc_empty__error"]) == "ZeroDivisionError"
    assert {G[f"{n}__logits"].shape[2] for n in ctc} == {32, 2599}
    # cv: the inf batch and the NaN batch are skipped, so the totals are finite
    assert np.isfinite(G["cv_ctc__loss"]) and np.isfinite(G["cv_mp__loss"])
    assert np.isinf(G["ctc0__loss"]) and G["cv_ctc_b0__feats"].shape == G["ctc0__logits"].shape


@pytest.mark.skipif(not have_reference(), reason="reference sources not present")
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_oracle_equals_live_reference(seed):
    import sys
    from tests.conftest import REFERENCE
    if REFERENCE not in sys.path:
        sys.path.insert(0, REFERENCE)
    from wekws.model.loss import criterion as ref
    gen = torch.Generator().manual_seed(seed)
    B, T, D = 9, 31, 3
    x = torch.rand(B, T, D, generator=gen) ** 2
    t = torch.randint(-2, D + 1, (B,), generator=gen)
    lens = torch.randint(1, T + 1, (B,), generator=gen)
    lens[0] = T
    for md in (0, 4):
        a, b = ref("max_pooling", x, t, lens, None, md), K.criterion("max_pooling", x, t, lens, None, md)
        assert float(a[0]) == float(b[0]) and a[1] == b[1]
    xc = torch.randn(B, 7, generator=gen) * 3
    tc = torch.randint(0, 7, (B,), generator=gen)
    tc[2] = -100
    a, b = ref("ce", xc, tc, None), K.criterion("ce", xc, tc, None)
    assert float(a[0]) == float(b[0]) and a[1] == b[1]
    V, T = 12, 30
    x = torch.randn(B, T, V, generator=gen) * 3
    tl = torch.randint(0, 6, (B,), generator=gen)
    tl[0] = 3
    tgt = torch.randint(1, V, (B, 5), generator=gen)
    tgt[torch.arange(5)[None, :] >= tl[:, None]] = -1
    lens = torch.randint(6, T + 1, (B,), generator=gen)
    for val in (False, True):
        a, b = ref("ctc", x, tgt, lens, tl, 0, val), K.criterion("ctc", x, tgt, lens, tl, 0, val)
        assert float(a[0]) == float(b[0]) and a[1] == b[1]


def test_device_criterion_refuses_cpu_input():
    from wekws_b200 import criterion
    x = torch.rand(2, 5, 2)
    with pytest.raises(ValueError):
        criterion("max_pooling", x, torch.tensor([0, -1]), torch.tensor([5, 5]))
    with pytest.raises(ValueError):
        criterion("ce", torch.randn(2, 3), torch.tensor([0, 1]), None)
    with pytest.raises(ValueError):
        criterion("ctc", torch.randn(2, 5, 4), torch.tensor([[1], [2]]), torch.tensor([5, 5]), torch.tensor([1, 1]))
    with pytest.raises(SystemExit):
        criterion("mse", x, torch.tensor([0, -1]), torch.tensor([5, 5]))
