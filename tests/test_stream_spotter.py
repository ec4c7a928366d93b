"""GPU tests of wekws_b200.KeywordSpotter: the streaming front-end against the reference's accept_wave
(tests/golden/spotter.npz) and the oracle, ctc_spot_kernel against the reference's decisions, and the whole spotter
end to end against the oracle restatement driven by the same model."""
import numpy as np
import pytest
import torch

from oracle.kws_spotter_oracle import SpotterOracle
from tests.conftest import golden
from tests.test_spotter_host import ScriptedProbs, case_pcm, decode_result, golden_case, golden_keywords
from wekws_b200 import Fbank, KeywordSpotter, _native, init_model, model_config, synth
from wekws_b200.ctc import SPOT_RESULT_DTYPE, CtcSpotDecoder

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _model(name, idim, odim, seed=3, scale=1.0):
    cfg = model_config(name, input_dim=idim, output_dim=odim, activation="identity")
    m = synth.randomize_(init_model(cfg), seed=seed).eval()
    last = "backbone.out_linear2.linear" if name == "fsmn" else "classifier.linear"
    with torch.no_grad():                  # sharper posteriors: a peaky CTC-like output
        m.get_submodule(last).weight.mul_(scale)
        m.get_submodule(last).bias.zero_()
    m.precision = "fp32"
    return m.to(DEV)


def _frontend_model(c, odim=48):
    if c["context"]:
        return Fbank(c["mel"]), _model("fsmn", c["mel"] * 5, odim)
    return Fbank(c["mel"]), _model("ds_tcn", c["mel"], odim)


def test_frontend_matches_reference_and_oracle():
    """Per golden chunk: the frame count the reference's accept_wave produced, its features within the Fbank gate,
    and the context / skip rows bit-exact with the oracle applied to the device's own Fbank rows."""
    g = golden("spotter")
    kws = golden_keywords(g)
    for i in range(int(g["ncases"])):
        c = golden_case(g, i)
        fb, model = _frontend_model(c)
        spot = KeywordSpotter(model, kws, 1, frontend=fb, context=c["context"], frame_skip=c["skip"])
        dev_rows = {}
        o = SpotterOracle(kws, lambda f: torch.zeros(f.shape[0], 48), num_mel_bins=c["mel"], context=c["context"],
                          frame_skip=c["skip"], fbank=lambda w: dev_rows["f"])
        lens = g[f"lens{i}"]
        pcm = torch.from_numpy(case_pcm(int(g[f"seed{i}"]), int(lens.sum())))
        pos, fpos = 0, 0
        for k, n in enumerate(lens):
            chunk = torch.zeros(1, max(int(n), 1), dtype=torch.int16)
            chunk[0, :n] = pcm[pos:pos + n]
            res = spot(chunk.to(DEV), [int(n)])
            frames = int(g[f"frames{i}"][k])
            assert int(res.frames[0]) == max(frames, 0), (i, k)
            dev_rows["f"] = res.fbank_rows(0).cpu()
            want = o.accept_wave(pcm[pos:pos + n].numpy())
            pos += n
            x = res.model_input(0).cpu()
            if want is None or want.shape[0] == 0:
                assert int(res.frames[0]) == 0
                continue
            assert torch.equal(x, want), (i, k)                      # copies only: bit-exact
            if k < int(g["feat_chunks"]):
                ref = g[f"feats{i}"][fpos:fpos + x.shape[0]]
                fpos += x.shape[0]
                d = np.abs(x.numpy() - ref)
                assert d.max() <= 1e-3 and d.mean() <= 1e-5, (i, k, d.max(), d.mean())
        assert fpos == len(g[f"feats{i}"])


def _golden_decoder(g, i, B):
    c = golden_case(g, i)
    return CtcSpotDecoder(B, golden_keywords(g), 3, 20, c["skip"], c["threshold"], c["min_frames"], c["max_frames"],
                          c["interval_frames"], DEV)


def _check_hyps(got, g, i):
    n = len(g[f"hyp_len{i}"])
    assert len(got) == n
    for j, (prefix, score, nodes) in enumerate(got):
        L = int(g[f"hyp_len{i}"][j])
        assert list(prefix) == g[f"hyp_tok{i}"][j, :L].tolist()
        assert [nd["frame"] for nd in nodes] == g[f"hyp_frame{i}"][j, :L].tolist()
        assert [nd["prob"] for nd in nodes] == g[f"hyp_prob{i}"][j, :L].tolist()
        assert score == float(g[f"hyp_pb{i}"][j]) + float(g[f"hyp_pnb{i}"][j])


@pytest.mark.parametrize("B", [1, 1000])
def test_spot_kernel_matches_reference_golden(B):
    """The reference's probabilities through ctc_spot_kernel: every return value and the final hypotheses are
    bit-exact, no overflow.  B = 1000: the golden stream replicated, each copy at a permuted row of the buffer."""
    g = golden("spotter")
    words = [str(w) for w in g["kw_names"]]
    perm_rng = np.random.RandomState(B)
    for i in range(int(g["ncases"])):
        dec = _golden_decoder(g, i, B)
        probs = torch.from_numpy(g[f"probs{i}"])
        pos = 0
        for k, T in enumerate(g[f"frames{i}"]):
            want = decode_result(g[f"result{i}"][k], words)
            if T <= 0:
                assert want == {}
                continue
            T = int(T)
            perm = perm_rng.permutation(B)
            buf = probs[pos:pos + T].repeat(B, 1).to(DEV)            # slot s holds rows s*T .. s*T + T-1
            rows = torch.tensor(perm * T, dtype=torch.int32, device=DEV)
            frames = torch.full((B,), T, dtype=torch.int32, device=DEV)
            pos += T
            raw = dec(buf, rows, frames).cpu().numpy().view(SPOT_RESULT_DTYPE).reshape(B)
            assert (raw["overflow"] == 0).all()
            for b in range(B) if B == 1 else (0, B // 2, B - 1):
                r = raw[b]
                got = ({"state": 1, "keyword": words[r["keyword"]], "start": int(r["start"]) * 0.01,
                        "end": int(r["end"]) * 0.01, "score": float(r["score"])} if r["state"] == 1 else
                       {"state": 0, "keyword": None, "start": None, "end": None, "score": None})
                assert got == {k2: (None if v != v else v) for k2, v in want.items()}, (i, k, b)
            for f in ("state", "keyword", "start", "end", "score"):
                assert (raw[f] == raw[f][0]).all()
        hyps = dec.hypotheses()
        for b in range(B) if B == 1 else (0, B - 1):
            _check_hyps(hyps[b], g, i)


class _PerStream:
    """The oracle's model step: the same KWSModel, one stream, softmax fused, its own cache."""

    def __init__(self, model):
        self.model, self.cache = model, None

    def __call__(self, feats):
        y, self.cache = self.model.forward_softmax(feats.unsqueeze(0).to(DEV),
                                                   self.cache if self.cache is not None else torch.zeros(0, 0, 0))
        return y[0].cpu()

    def reset(self):
        self.cache = None


def _emitted_tokens(model, fb, ctx, skip, n=3):
    """The n most frequent non-blank arg-max tokens of the model on a sample of the test audio."""
    pcm = synth.pcm_int16(4, 16000, seed=77).to(DEV)
    f = fb(pcm)
    if ctx:
        from wekws_b200 import context_expansion
        f, _ = context_expansion(f, ctx[0], ctx[1], skip)
    y, _ = model.forward_softmax(f.contiguous())
    counts = torch.bincount(y.argmax(-1).flatten().cpu(), minlength=model.odim)
    counts[0] = 0
    return counts.argsort(descending=True)[:n].tolist()


@pytest.mark.parametrize("name", ["fsmn", "ds_tcn"])
@pytest.mark.parametrize("B", [1, 257])
def test_spotter_end_to_end_matches_oracle(name, B):
    """Mixed chunk lengths (zero-length chunks too) and reset() of some streams mid-run, so that several groups form
    in one call.  Every result equals the oracle restatement driven by the same FP32 KWSModel run per stream on the
    spotter's own features."""
    ctx, skip, mel = ((2, 2), 3, 80) if name == "fsmn" else (None, 1, 40)
    fb = Fbank(mel)
    model = _model(name, mel * (5 if ctx else 1), 24, seed=5, scale=12.0)
    a, b, c = _emitted_tokens(model, fb, ctx, skip)
    kws = {"k_ab": [a, b], "k_bc": [b, c], "k_ca": [c, a]}
    params = dict(threshold=0.0, min_frames=5, max_frames=100, interval_frames=20)
    spot = KeywordSpotter(model, kws, B, frontend=fb, context=ctx, frame_skip=skip, **params)
    oracles = [SpotterOracle(kws, _PerStream(model), num_mel_bins=mel, context=ctx, frame_skip=skip,
                             fbank=None, **params) for _ in range(B)]
    rows = {}
    for o in oracles:
        o.fbank = lambda w, o=o: rows[id(o)]
    rng = np.random.RandomState(B + len(name))
    nchunks = 24 if B == 1 else 12
    audio = synth.pcm_int16(B, 6000 * nchunks, seed=B)
    premise_checked = False
    activations, groups_seen = 0, 0
    for k in range(nchunks):
        if k in (nchunks // 3, 2 * nchunks // 3):
            who = sorted(rng.choice(B, size=max(1, B // 5), replace=False).tolist())
            spot.reset(who)
            for s in who:
                oracles[s].reset_all()
        lens = [int(rng.choice([4800, 4800, 4800, 0, int(rng.randint(0, 6000)), int(rng.randint(0, 900))]))
                for _ in range(B)]
        chunk = audio[:, k * 6000:(k + 1) * 6000].to(DEV)
        res = spot(chunk, lens)
        groups_seen = max(groups_seen, len(set(res.frames[res.frames > 0].tolist())))
        if not premise_checked and (res.frames > 0).any():
            # premise: the FP32 forward is bitwise the same per stream and batched (B = 1: the stream twice)
            T = int(res.frames[res.frames > 0][0])
            idx = ([s for s in range(B) if res.frames[s] == T] * 2)[:8]
            x = torch.stack([res.model_input(s) for s in idx])
            yb, _ = model.forward_softmax(x.contiguous())
            for j in range(len(idx)):
                y1, _ = model.forward_softmax(x[j:j + 1].contiguous())
                assert torch.equal(y1[0], yb[j]), "premise failed: FP32 forward differs per stream vs batched"
            premise_checked = True
        got = res.to_python()
        assert (res.overflow == 0).all()
        for s in range(B):
            rows[id(oracles[s])] = res.fbank_rows(s).cpu()
            want = oracles[s].forward(chunk[s, :lens[s]].cpu().numpy(), feats=res.model_input(s).cpu()
                                      if res.frames[s] > 0 else None)
            assert got[s] == want, (name, B, k, s, got[s], want)
            activations += int(got[s].get("state", 0) == 1)
    assert premise_checked
    if B > 1:
        assert groups_seen >= 2
    test_spotter_end_to_end_matches_oracle.activations[(name, B)] = activations


test_spotter_end_to_end_matches_oracle.activations = {}


def test_end_to_end_activations_not_vacuous():
    acts = test_spotter_end_to_end_matches_oracle.activations
    if len(acts) < 4:
        pytest.skip("runs after the end-to-end tests")
    assert sum(acts.values()) >= 20, acts


def test_steady_state_launch_count():
    """One group (every stream, same chunk length): PCM, Fbank, context, the model's own launches, spot."""
    B = 64
    fb = Fbank(80)
    model = _model("fsmn", 400, 48)
    spot = KeywordSpotter(model, {"a": [5, 9, 17]}, B, frontend=fb, context=(2, 2), frame_skip=3)
    pcm = synth.pcm_int16(B, 4800, seed=3).to(DEV)
    for _ in range(3):
        spot(pcm)
    torch.cuda.synchronize()
    x = torch.randn(B, 10, 400, device=DEV)
    n0 = _native.launch_count()
    model.forward_softmax(x)
    torch.cuda.synchronize()
    model_launches = _native.launch_count() - n0
    n0 = _native.launch_count()
    fb(pcm)
    torch.cuda.synchronize()
    fbank_launches = _native.launch_count() - n0
    counts = []
    for _ in range(4):
        n0 = _native.launch_count()
        res = spot(pcm)
        counts.append(_native.launch_count() - n0)
        assert len(set(res.frames.tolist())) == 1
    assert counts == [1 + fbank_launches + 1 + model_launches + 1] * 4, (counts, fbank_launches, model_launches)


def test_spotter_refuses_bad_input():
    model = _model("fsmn", 400, 48)
    spot = KeywordSpotter(model, {"a": [5, 9]}, 4, frontend=Fbank(80), context=(2, 2), frame_skip=3)
    pcm = torch.zeros(4, 100, dtype=torch.int16, device=DEV)
    with pytest.raises(ValueError):
        spot(pcm.float())
    with pytest.raises(ValueError):
        spot(pcm[:3])
    with pytest.raises(ValueError):
        spot(pcm.cpu())
    with pytest.raises(ValueError):
        spot(pcm, [0, 1, 2, 101])
    with pytest.raises(ValueError):
        spot(pcm, [0, 1, 2])
    with pytest.raises(ValueError):
        spot.reset([4])
    assert spot(pcm, [0, 0, 0, 0]).to_python() == [{}] * 4
