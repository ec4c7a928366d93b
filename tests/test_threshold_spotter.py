"""GPU tests of wekws_b200.ThresholdSpotter / ThresholdDecoder: threshold_spot_kernel against the stats files the
reference's compute_det.py wrote (tests/golden/det_stats.npz) in random chunkings, the rule's edges, every max-pooling
recipe end to end against the whole-utterance model and det_stats, stream permutation and reset, and the launches of a
steady-state call."""
import numpy as np
import pytest
import torch

from tests.conftest import golden
from tests.test_threshold_spotter_host import RECIPE_FEATURES, OnlineRule, random_chunks
from wekws_b200 import (Fbank, KeywordSpotter, Mfcc, ThresholdDecoder, ThresholdSpotter, _native, det_curve, det_stats,
                        det_thresholds, init_model, model_config, synth)
from wekws_b200.spotter import trained_front_end

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _feed(dec, chunks, K, perm=None):
    """Runs `dec` over one call per entry of `chunks` (per call, per stream, its (n, K) rows; None = no frames), the
    streams' rows placed in the order `perm`.  Returns per stream its events [(frame, keyword, score)] in call order."""
    B = dec.B
    perm = np.arange(B) if perm is None else perm
    out = [[] for _ in range(B)]
    for call in chunks:
        n = np.array([0 if c is None else len(c) for c in call])
        rows = np.zeros(B, np.int64)
        base = 0
        for b in perm:
            rows[b] = base
            base += n[b]
        probs = np.zeros((max(base, 1), K), np.float32)
        for b in range(B):
            if n[b]:
                probs[rows[b]:rows[b] + n[b]] = call[b]
        buf = dec(torch.from_numpy(probs).to(DEV), torch.tensor(rows, dtype=torch.int32, device=DEV),
                  torch.tensor(n, dtype=torch.int32, device=DEV))
        counts, events = dec.unpack(buf)
        assert events.shape[2] == -(-int(n.max()) // dec.window_shift)
        for b in range(B):
            for k in range(K):
                out[b] += [(int(e["frame"]), int(e["keyword"]), float(e["score"])) for e in events[b, k, :counts[b, k]]]
    return out


def _golden_calls(post, lens, ws, rng):
    """Each utterance in its own random chunking (empty and one-frame chunks included), one call per chunk index."""
    B = post.shape[0]
    sizes = [random_chunks(rng, int(lens[b]), ws) for b in range(B)]
    ncalls = max(len(s) for s in sizes)
    calls, pos = [], [0] * B
    for i in range(ncalls):
        call = []
        for b in range(B):
            s = sizes[b][i] if i < len(sizes[b]) else 0
            call.append(post[b, pos[b]:pos[b] + s] if s else None)
            pos[b] += s
        calls.append(call)
    return calls


def test_decoder_reproduces_reference_compute_det_files():
    """One ThresholdDecoder per threshold of the sweep, the golden posteriors in random chunkings: the firings per
    utterance, through det_curve, give the stats files the reference's compute_det.py wrote, text for text.  A keyword
    utterance is a false reject at x when it never fires at x (max score < x), so its max score enters det_curve as the
    largest threshold at which it fired."""
    g = golden("det_stats")
    post, lens = g["post"], g["lens"]
    B, T, K = post.shape
    kinds, durs = g["kinds"].tolist(), g["durations"].tolist()
    rng = np.random.RandomState(17)
    for si, (ws, step) in enumerate(g["settings"].tolist()):
        ws = int(ws)
        thr = det_thresholds(step)
        calls = _golden_calls(post, lens, ws, rng)
        triggers = torch.zeros(B, K, thr.numel(), dtype=torch.int32)
        for i, th in enumerate(thr.tolist()):
            ev = _feed(ThresholdDecoder(B, [th] * K, ws, DEV), calls, K, perm=rng.permutation(B))
            for b in range(B):
                for _, k, _ in ev[b]:
                    triggers[b, k, i] += 1
        _, _, want = det_stats(torch.from_numpy(post).to(DEV), torch.from_numpy(lens).to(DEV), step=step,
                               window_shift=ws)
        assert torch.equal(triggers, want.cpu()), si
        fired = triggers > 0
        max_score = torch.where(fired.any(-1), (thr * fired).max(-1).values, torch.tensor(-float("inf"),
                                                                                           dtype=torch.float64))
        for k in range(K):
            filler = 0.0
            for b, kd in enumerate(kinds):
                if kd != k:
                    filler += durs[b]
            rows = det_curve(thr, max_score, triggers, [kd == k for kd in kinds], filler_hours=filler / 3600.0,
                             keyword_index=k)
            text = "".join("{:.6f} {:.6f} {:.6f}\n".format(*r) for r in rows)
            assert text == str(g[f"stats_{si}_{k}"]), (si, k)


def _one(dec, *chunks):
    """One stream, one keyword: the frames that fired in each chunk."""
    return [[e[0] for e in _feed(dec, [[np.asarray(c, np.float32).reshape(-1, 1) if len(c) else None]], 1)[0]]
            for c in chunks]


def test_rule_edges():
    # a firing on a chunk's last frame suppresses the next window_shift - 1 frames, in later chunks
    dec = ThresholdDecoder(1, [0.5], 4, DEV)
    assert _one(dec, [0.1, 0.9], [0.9, 0.9], [], [0.9], [0.9, 0.9]) == [[1], [], [], [], [5]]
    # window_shift 1: every frame at or above the threshold fires
    dec = ThresholdDecoder(1, [0.5], 1, DEV)
    assert _one(dec, [0.9, 0.9, 0.2], [0.7], [0.5, 0.49]) == [[0, 1], [3], [4]]
    # threshold 0 fires every window_shift frames, whatever the chunking
    dec = ThresholdDecoder(1, [0.0], 3, DEV)
    assert sum(_one(dec, [0.0] * 4, [0.0], [0.0] * 2, [], [0.0] * 6), []) == [0, 3, 6, 9, 12]
    # the 6-decimal text rounding: both print as 0.500000, as '{:.6f}' does
    x = [0.4999995, 0.5000005, 0.4999994, 0.5]
    want = [t for t, v in enumerate(x) if float('{:.6f}'.format(np.float32(v))) >= 0.5]
    dec = ThresholdDecoder(1, [0.5], 1, DEV)
    assert sum(_one(dec, x[:1], x[1:]), []) == want == OnlineRule(0.5, 1)(np.array(x, np.float32))
    assert 1 in want
    # frame indices past 2^31: the record (seen, next) is two int64 (include/wekws_b200.h)
    dec = ThresholdDecoder(2, [0.0], 2, DEV)
    rec = dec.state.view(torch.int64).view(2, 1, 2)
    rec[1, 0, 0] = 2 ** 31 - 3
    rec[1, 0, 1] = 2 ** 31 - 2
    ev = _feed(dec, [[np.zeros((3, 1), np.float32), np.zeros((6, 1), np.float32)]], 1)
    assert [e[0] for e in ev[0]] == [0, 2]
    assert [e[0] for e in ev[1]] == [2 ** 31 - 2, 2 ** 31, 2 ** 31 + 2]
    assert rec[1, 0].tolist() == [2 ** 31 + 3, 2 ** 31 + 4]
    ev = _feed(dec, [[None, np.zeros((2, 1), np.float32)]], 1)
    assert [[e[0] for e in x] for x in ev] == [[], [2 ** 31 + 4]]      # frame 2^31 + 3 is suppressed


# every max-pooling recipe shipped: (recipe, model_config name, model input width, outputs, hidden_dim override)
RECIPES = [("hi_xiaowen/mdtc", "mdtc", 80, 2, None), ("hi_xiaowen/mdtc_small", "mdtc_small", 80, 2, None),
           ("hi_xiaowen/ds_tcn", "ds_tcn", 40, 2, None), ("hi_xiaowen/tcn", "tcn", 40, 2, None),
           ("hi_xiaowen/gru", "gru", 40, 2, None), ("hey_snips/ds_tcn", "ds_tcn", 40, 1, 64),
           ("hey_snips/mdtc_small", "mdtc_small", 80, 1, None)]


def _recipe_model(name, mel, odim, hidden, seed=5):
    cfg = model_config(name, input_dim=mel, output_dim=odim)
    if hidden:
        cfg["hidden_dim"] = hidden
    m = synth.randomize_(init_model(cfg), seed=seed).eval()
    m.precision = "fp32"
    return m.to(DEV)


def _stream_audio(B, rng):
    lens = rng.randint(4800, 48001, size=B)                  # 0.3 .. 3 s
    return [synth.pcm_int16(1, int(n), seed=int(rng.randint(1 << 30)))[0] for n in lens]


def _chunk_plan(audio, rng):
    """Per call, per stream, a chunk length: empty, shorter than one window, or up to 0.6 s, until all is sent."""
    pos, plan = [0] * len(audio), []
    while any(p < len(a) for p, a in zip(pos, audio)):
        lens = []
        for b, a in enumerate(audio):
            n = int(rng.choice([0, int(rng.randint(1, 400)), int(rng.randint(400, 9600)), int(rng.randint(1, 9600))]))
            n = min(n, len(a) - pos[b])
            lens.append(n)
            pos[b] += n
        plan.append(lens)
    return plan


def _run(spot, audio, plan, order=None):
    """Feeds the plan; returns per stream (its firings [(frame, keyword index, score)], its posteriors (F, K) on the
    host), stream b of the result being audio[order[b]]."""
    B = len(audio)
    order = list(range(B)) if order is None else order
    pos = [0] * B
    events, posts = [[] for _ in range(B)], [[] for _ in range(B)]
    for lens in plan:
        lens = [lens[order[b]] for b in range(B)]
        N = max(max(lens), 1)
        pcm = torch.zeros(B, N, dtype=torch.int16)
        for b in range(B):
            a = audio[order[b]]
            pcm[b, :lens[b]] = a[pos[b]:pos[b] + lens[b]]
            pos[b] += lens[b]
        res = spot(pcm.to(DEV), lens)
        for b in range(B):
            posts[b].append(res.posteriors(b).cpu())
            for e in res.to_python()[b]:
                events[b].append((e["frame"], spot.words.index(e["keyword"]), e["score"]))
                assert e["time"] == e["frame"] * spot.frame_seconds
    return events, [torch.cat(p) if p else torch.zeros(0, spot.decoder.K) for p in posts]


@pytest.mark.parametrize("recipe", RECIPES, ids=[r[0] for r in RECIPES])
def test_end_to_end_every_max_pooling_recipe(recipe):
    """Each recipe through from_config with its own dataset_conf feature section (MFCC for mdtc / mdtc_small), streams
    of their own lengths in random chunks.  Each stream fires exactly where the host scan of its own posteriors fires;
    at precision fp32 its concatenated posteriors are bit for bit those of the model run once over the recipe's
    front-end on the whole utterance, so its firings are det_stats' triggers on the whole utterance."""
    key, name, idim, odim, hidden = recipe
    model = _recipe_model(name, idim, odim, hidden)
    conf = {"dataset_conf": RECIPE_FEATURES[key]}
    fe = trained_front_end(conf)[0]
    assert isinstance(fe, Mfcc) == name.startswith("mdtc")
    rng = np.random.RandomState(len(key))
    B = 6
    audio = _stream_audio(B, rng)
    whole = []
    for a in audio:
        y, _ = model(fe(a.to(DEV).unsqueeze(0)))
        whole.append(y[0].cpu())
    allp = torch.cat(whole)
    thr = [float(np.quantile(allp[:, k].numpy(), 0.9)) for k in range(odim)]     # a threshold that fires
    ws = 7
    spot = ThresholdSpotter.from_config(conf, model, B, thresholds=thr, window_shift=ws,
                                        keywords=[f"kw{k}" for k in range(odim)])
    assert type(spot.front.frontend) is type(fe)
    events, posts = _run(spot, audio, _chunk_plan(audio, rng))
    fired = 0
    for b in range(B):
        assert torch.equal(posts[b], whole[b]), (key, b, (posts[b] - whole[b]).abs().max())
        want = sorted((t, k, float(posts[b][t, k])) for k in range(odim)
                      for t in OnlineRule(thr[k], ws)(posts[b][:, k].numpy()))
        assert events[b] == want, (key, b)
        fired += len(events[b])
        for k in range(odim):
            assert sum(1 for e in events[b] if e[1] == k) == _det_triggers(whole[b][:, k], thr[k], ws)
    assert fired > 0


def _det_triggers(post, th, ws):
    """wekws_det_stats' trigger count of one posterior track at the single threshold th."""
    p = post.contiguous().view(1, -1, 1).to(DEV)
    ms = torch.empty(1, 1, dtype=torch.float64, device=DEV)
    tr = torch.empty(1, 1, 1, dtype=torch.int32, device=DEV)
    _native.call("wekws_det_stats", p, None, 1, p.shape[1], 1, torch.tensor([th], dtype=torch.float64, device=DEV), 1,
                 ws, ms, tr, device=torch.device(DEV))
    return int(tr.item())


def test_permutation_and_reset():
    """Permuting the streams permutes their firings; reset([b]) and then audio fires as a fresh spotter does."""
    model = _recipe_model("ds_tcn", 40, 2, None)
    fb = Fbank(40)
    rng = np.random.RandomState(3)
    B = 5
    audio = _stream_audio(B, rng)
    y, _ = model(fb(audio[0].to(DEV).unsqueeze(0)))
    thr = [float(np.quantile(y[0, :, k].cpu().numpy(), 0.8)) for k in range(2)]
    plan = _chunk_plan(audio, rng)
    ev_a, post_a = _run(ThresholdSpotter(model, thr, B, frontend=fb, window_shift=5), audio, plan)
    order = [3, 0, 4, 1, 2]
    ev_b, post_b = _run(ThresholdSpotter(model, thr, B, frontend=fb, window_shift=5), audio, plan, order)
    for b in range(B):
        assert ev_b[b] == ev_a[order[b]] and torch.equal(post_b[b], post_a[order[b]])
    assert sum(len(e) for e in ev_a) > 0
    # stream 2 hears other audio first, is reset, then hears audio[2]: it fires as a fresh spotter on audio[2] does
    spot = ThresholdSpotter(model, thr, B, frontend=fb, window_shift=5)
    noise = [synth.pcm_int16(1, 30000, seed=99)[0] for _ in range(B)]
    _run(spot, noise, _chunk_plan(noise, rng))
    spot.reset([2])
    ev_r, post_r = _run(spot, audio, plan)
    assert ev_r[2] == ev_a[2] and torch.equal(post_r[2], post_a[2])


def test_steady_state_launches_and_determinism():
    """One group (every stream, same chunk length): PCM, Fbank, context rows, the model's own launches, detection;
    one host-to-device table and one device-to-host result per call.  Repeated runs give the same results."""
    B = 64
    fb = Fbank(40)
    model = _recipe_model("ds_tcn", 40, 2, None)
    pcm = synth.pcm_int16(B, 8000 * 6, seed=3).to(DEV)
    chunks = [pcm[:, i * 8000:(i + 1) * 8000] for i in range(6)]
    spot = ThresholdSpotter(model, [0.3, 0.3], B, frontend=fb, window_shift=10)
    for c in chunks[:2]:
        spot(c)
    torch.cuda.synchronize()
    x = torch.randn(B, 50, 40, device=DEV)
    n0 = _native.launch_count()
    model(x)
    torch.cuda.synchronize()
    model_launches = _native.launch_count() - n0
    n0 = _native.launch_count()
    fb(chunks[0])
    torch.cuda.synchronize()
    fbank_launches = _native.launch_count() - n0
    counts = []
    for c in chunks[2:]:
        n0 = _native.launch_count()
        res = spot(c)
        counts.append(_native.launch_count() - n0)
        assert len(set(res.frames.tolist())) == 1 and res.frames[0] == 50
    assert counts == [1 + fbank_launches + 1 + model_launches + 1] * 4, (counts, fbank_launches, model_launches)
    runs = []
    for _ in range(2):
        s = ThresholdSpotter(model, [0.3, 0.3], B, frontend=fb, window_shift=10)
        runs.append([(r.counts.copy(), r.events.copy(), r.to_python()) for r in (s(c) for c in chunks)])
    for (c1, e1, p1), (c2, e2, p2) in zip(*runs):
        assert np.array_equal(c1, c2) and p1 == p2
        for b in range(B):                      # only the first counts[b, k] slots of each (b, k) are written
            for k in range(2):
                assert np.array_equal(e1[b, k, :c1[b, k]], e2[b, k, :c2[b, k]])
    assert sum(int(c.sum()) for c, _, _ in runs[0]) > 0


def test_spotter_refuses_bad_input():
    model = _recipe_model("ds_tcn", 40, 2, None)
    spot = ThresholdSpotter(model, [0.5, 0.5], 4, frontend=Fbank(40))
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
        spot(pcm, torch.tensor([0, 1, 2, 3], device=DEV))
    with pytest.raises(ValueError):
        spot.reset([4])
    res = spot(pcm, [0, 0, 0, 0])
    assert res.to_python() == [[]] * 4 and res.counts.shape == (4, 2) and res.posteriors(0).shape == (0, 2)


def test_decoder_refuses_bad_tables():
    """The standalone decoder checks its tables; a max_frames below the largest frame count cannot drop events
    silently."""
    dec = ThresholdDecoder(2, [0.0], 1, DEV)
    probs = torch.zeros(5, 1, device=DEV)
    rows = torch.tensor([0, 3], dtype=torch.int32, device=DEV)
    frames = torch.tensor([3, 2], dtype=torch.int32, device=DEV)
    for bad in (rows.long(), rows.cpu(), rows[:1], torch.stack([rows, rows], 1)[:, 0]):
        with pytest.raises(ValueError, match="rows must be"):
            dec(probs, bad, frames)
    with pytest.raises(ValueError, match="frames must be"):
        dec(probs, rows, frames.float())
    with pytest.raises(ValueError, match="lie in the 5 rows"):
        dec(probs, rows, torch.tensor([3, 3], dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="lie in the 5 rows"):
        dec(probs, torch.tensor([-1, 3], dtype=torch.int32, device=DEV), frames)
    with pytest.raises(ValueError, match="probs must be"):
        dec(probs[:0], rows, torch.zeros(2, dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError, match="outputs per row"):
        dec(torch.zeros(5, 2, device=DEV), rows, frames)
    assert dec.state.abs().sum() == 0                       # nothing ran
    with pytest.raises(RuntimeError, match="max_frames was below"):
        dec.unpack(dec(probs, rows, frames, max_frames=1))  # threshold 0, window 1: 3 firings, 1 slot
    counts, events = dec.unpack(dec(probs, rows, frames))
    assert counts.tolist() == [[3], [2]] and events["frame"][0, 0].tolist() == [3, 4, 5]


def test_keyword_spotter_keeps_its_attributes():
    """model, frontend, cache and mirror are still reachable on KeywordSpotter after the front half moved out."""
    cfg = model_config("ds_tcn", input_dim=40, output_dim=24, activation="identity")
    model = synth.randomize_(init_model(cfg), seed=3).eval().to(DEV)
    fb = Fbank(40)
    spot = KeywordSpotter(model, {"a": [1, 2]}, 3, frontend=fb)
    assert spot.model is model and spot.frontend is fb and spot.mirror is spot.front.mirror
    assert spot.cache is spot.front.cache and tuple(spot.cache.shape) == tuple(model.cache_shape(3))
