"""The backbone kernels at the batch sizes and chunk heights that select their other launch partitions.

Every forward kernel splits its work at launch from the batch B, the chunk height T and the SM count: streams per
tile and per pass, passes and tiles per CTA, landing-slot shares.  tests/test_config_sweep.py covers the model
configurations at B <= 300; here the same rows (and the shipped shapes) run at the batches and chunk heights where
the other branches of those partitions execute:

    gru_tc.cu      16 / 32 / 64 streams per tile, two tiles on one CTA, a partial last tile
    gru.cu         2 / 4 / 8 streams per CTA, two tiles on one CTA
    linear_tc.cu   two 128-row M tiles on one CTA, a partial M tile, a 39-column N tail (V = 2599)
    mdtc_tc.cu     1, 2 and >= 3 passes per CTA, a last pass of one tile, more streams than landing slots, passes
                   bounded by the X columns (chunks of 9..16 frames), one stream over both warpgroups (128 frames);
                   the `global` / `last` head variant with 16 streams per tile, several passes and several chunks
    tcn_tc.cu      the same pass structure, and one stream per pass (receptive field 448)
    dstcn_tc.cu    several passes per CTA at chunk heights 8, 60, 61 and 120
    conv_backbone.cu (FP32) T < 8 for 1024 streams

Without a GPU: `partition` restates each kernel's launch partition from the constants it reads out of the CUDA
sources, and a test checks that the GPU cases below reach every class in REQUIRED for 132 and 114 SMs.  The table
only chooses and checks shapes; it is never the reference for values.  On the GPU every case runs once from a random
cache and once from none, and every stream's output and returned cache is compared with the float64 oracle
(oracle/kws_head_oracle.py: run on the device for the convolutional models, whose float64 convolutions are slow on
the host, on the host for the GRU) under the sweep's gates.  `-s` prints each case's error next to its gate.
"""
import os
import re
from collections import namedtuple

import pytest
import torch

from oracle import kws_head_oracle as HO
from tests.head_cases import HEAD_CASES, build_head_model, head_config
from tests.test_config_sweep import _ROW, _config, _gate, build_config, build_row, inputs
from wekws_b200 import init_model

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "wekws_b200", "csrc")


# ----------------------------------------------------------------------------------------- the launch partitions
def _cdiv(a, b):
    return -(-a // b)


def _ints(src, pattern):
    m = re.search(pattern, src)
    assert m, f"pattern not found in the kernel source: {pattern}"
    return [int(g) for g in m.groups()]


_CONSTS = None


def kernel_constants():
    """The partition constants of each kernel, read from its source: a change there moves the shapes below with it,
    or fails the coverage test, instead of silently leaving a branch untested."""
    global _CONSTS
    if _CONSTS is None:
        def src(name):
            with open(os.path.join(CSRC, name)) as f:
                return f.read()
        md, tc, ds, gt, gf, lt = (src(f) for f in ("mdtc_tc.cu", "tcn_tc.cu", "dstcn_tc.cu", "gru_tc.cu", "gru.cu",
                                                    "linear_tc.cu"))

        def const(s, name):
            return _ints(s, rf"constexpr int [^;]*\b{name} = (\d+)[,;]")[0]
        _CONSTS = dict(
            mdtc=dict(NG=const(md, "NG"), XCOLS=const(md, "XCOLS"), NSLOT=const(md, "NSLOT"),
                      NSLOT_HEAD=const(md, "NSLOT_HEAD"), POOL_SPT=const(md, "POOL_SPT"),
                      ROWS=_ints(md, r"a\.spt = (\d+) / a\.T;")[0],
                      MAXT=_ints(md, r"int tc_max_T\(\) \{ return (\d+); \}")[0]),
            tcn=dict(NTILE=const(tc, "NTILE"), XCOLS=const(tc, "XCOLS"), RPX=const(tc, "RPX"),
                     ROWS=_ints(tc, r"a\.spt = (\d+) / a\.T;")[0],
                     MAXT=_ints(tc, r"return room < (\d+) \? room : \d+;")[0]),
            dstcn=dict(RPX=const(ds, "RPX")),
            # ms = B > a sms ? ms_a : B > b sms ? ms_b : ms_c
            gru_tc=_ints(gt, r"a\.ms = a\.B > (\d+) \* sms0 \? (\d+) : a\.B > (\d+) \* sms0 \? (\d+) : (\d+);"),
            # S = B <= sms ? s1 : B <= a sms ? s2 : B <= b sms ? s4 : s8
            gru=_ints(gf, r"S = a\.B <= sms \? (\d+) : a\.B <= (\d+) \* sms \? (\d+) : a\.B <= (\d+) \* sms \? (\d+) "
                          r": (\d+);"),
            linear_tc=_ints(lt, r"a\.n_mtiles = \(int\)\(\(a\.rows \+ (\d+)\) / (\d+)\);")[1],
        )
        c = _CONSTS["tcn"]
        assert c["XCOLS"] <= c["RPX"]
    return _CONSTS


def _cta_streams(B, grid):
    """The distinct stream counts of the balanced contiguous partition the conv kernels make over their grid."""
    return sorted({B * (i + 1) // grid - B * i // grid for i in range(grid)})


def _passes(n, smax):
    """Streams of each pass of a CTA with n streams: as few passes as smax allows, balanced."""
    out = []
    while n > 0:
        ns = _cdiv(n, _cdiv(n, smax))
        out.append(ns)
        n -= ns
    return out


def _slot_shares(ns, spt, nslot):
    """mdtc_tc.cu loader_role: the landing slots of each tile of a pass of ns streams."""
    ntile, used, shares = _cdiv(ns, spt), 0, []
    for t in range(ntile):
        n_t = min(spt, ns - t * spt)
        want = n_t if ns <= nslot else max(1, nslot * n_t // ns)
        want = min(want, nslot - used - (ntile - 1 - t))
        shares.append(want)
        used += want
    return shares


def partition(kernel, B, T, padmax, sms, head=False):
    """The launch partition of one forward call of B streams x T frames: a dict per kernel (see the sources)."""
    K = kernel_constants()
    if kernel == "gru_tc":
        a, ms_a, b, ms_b, ms_c = K["gru_tc"]
        ms = ms_a if B > a * sms else ms_b if B > b * sms else ms_c
        tiles = _cdiv(B, ms)
        return dict(ms=ms, tiles=tiles, tiles_per_cta=_cdiv(tiles, min(tiles, sms)), partial=B % ms != 0)
    if kernel == "gru":
        s1, a, s2, b, s4, s8 = K["gru"]
        S = s1 if B <= sms else s2 if B <= a * sms else s4 if B <= b * sms else s8
        tiles = _cdiv(B, S)
        return dict(S=S, tiles=tiles, tiles_per_cta=_cdiv(tiles, min(tiles, sms)))
    if kernel == "linear_tc":
        rows, tile = B * T, K["linear_tc"]
        mt = _cdiv(rows, tile)
        return dict(m_tiles=mt, tiles_per_cta=_cdiv(mt, min(mt, sms)), partial=rows % tile != 0)
    # conv kernels: the call is cut into equal chunks of at most the kernel's height (model_host.cu)
    padr = (padmax + 3) & ~3
    maxT = dict(mdtc=K["mdtc"]["MAXT"], tcn=min(K["tcn"]["MAXT"], K["tcn"]["XCOLS"] - padr),
                dstcn=K["dstcn"]["RPX"])[kernel]
    nchunk = _cdiv(T, maxT)
    Tc = _cdiv(T, nchunk)
    if kernel == "dstcn":
        spt = K["dstcn"]["RPX"] // Tc
        smax, ntiles, grid = spt, 1, min(_cdiv(B, spt), sms)
    else:
        c = K[kernel]
        spt = c["ROWS"] // Tc
        ntiles = c["NG"] if kernel == "mdtc" else c["NTILE"]
        Lw = padr + (Tc if kernel == "mdtc" else (Tc + 3) & ~3)
        smax = min(ntiles * spt, c["XCOLS"] // Lw)
        grid = min(B, sms)
    nslot = K["mdtc"]["NSLOT_HEAD" if head else "NSLOT"]
    ctas = {}
    for n in _cta_streams(B, grid):
        ps = []
        for ns in _passes(n, smax):
            tiles = [min(spt, ns - i * spt) for i in range(_cdiv(ns, spt))]
            p = dict(ns=ns, tiles=tiles)
            if kernel == "mdtc":
                p["slots"] = _slot_shares(ns, spt, nslot)
                # live warpgroups of each tile: a tile of <= 64 rows leaves its second warpgroup idle (not the head)
                p["wgs"] = [1 if not head and n_t * Tc <= 64 else 2 for n_t in tiles]
            ps.append(p)
        ctas[n] = ps
    return dict(chunk=Tc, chunks=nchunk, spt=spt, smax=smax, x_bound=smax < ntiles * spt, ctas=ctas)


# ---------------------------------------------------------------------------------------------------- the cases
# model id -> (recipe, overrides) for the shipped shapes; ids of tests/test_config_sweep.py ROWS and of
# tests/head_cases.py HEAD_CASES name themselves
SHIPPED = {"mdtc": ("mdtc", {}), "tcn": ("tcn", {}), "ds_tcn": ("ds_tcn", {}), "gru": ("gru", {}),
           "ds_tcn_ctc": ("ds_tcn", dict(input_dim=40, output_dim=2599))}     # ds_tcn_ctc.yaml: V = 2599

# group: gru_tc / gru (FP32, precision "fp32"), conv (per-frame classifier, tensor cores), head, dstcn, linear (DS-TCN
# + linear_tc), conv32 (the FP32 conv kernel, T < 8).  batch: (k, r) = k sms + r streams, or "p1" / "p2" / "p3"
# (CTAs of p smax - 1 and p smax streams: p passes) or "tail" (CTAs of 2 spt + 1 streams: a two-tile pass, then a
# one-tile pass), resolved through `partition`.
Case = namedtuple("Case", "group model T batch")

_GRU_TC_B = [(16, 0), (16, 1), (32, 1), (64, 37)]
_GRU_B = [(1, 1), (2, 1), (4, 1), (8, 37)]
_CONV_T = {"mdtc": [9, 16, 17, 31, 64, 127, 128], "mdtc_1x1_i40_o3": [9, 16, 17, 31, 64, 127, 128],
           "tcn_k3x5_i40_o8": [9, 16, 17, 31, 64, 127, 128], "tcn_k8x7": [9, 16, 17, 31, 56]}
_TAIL_T = {"mdtc": [16, 128], "mdtc_1x1_i40_o3": [16, 31, 128], "tcn_k3x5_i40_o8": [16, 64]}


def _cases():
    cs = []
    for model in ("gru", "gru_1l_i40", "gru_i13"):
        cs += [Case("gru_tc", model, T, b) for b in _GRU_TC_B for T in (1, 3)]
        cs += [Case("gru", model, T, b) for b in _GRU_B for T in (1, 3)]
    for model, Ts in _CONV_T.items():
        cs += [Case("conv", model, T, p) for T in Ts for p in ("p1", "p2", "p3")]
        cs += [Case("conv", model, T, "tail") for T in _TAIL_T.get(model, [])]
    cs += [Case("dstcn", "dstcn_3l_i40_o4", T, p) for T in (8, 60, 61, 120) for p in ("p2", "p3")]
    for model in ("ds_tcn_ctc", "dstcn_4l_o128"):
        cs.append(Case("linear", model, 121, "linear"))
    for model in ("mdtc_2x3_i40_last", "mdtc_global", "mdtc_last", "tcn_global"):
        cs += [Case("head", model, T, b) for T in (8, 40, 128, 300) for b in ((1, 1), (4, 3))]
    for model in ("mdtc", "tcn", "ds_tcn"):
        cs += [Case("conv32", model, T, b) for T in (1, 4, 7) for b in ((0, 1024), (4, 3))]
    return cs


CASES = _cases()


def case_id(c):
    b = c.batch if isinstance(c.batch, str) else f"{c.batch[0]}sms+{c.batch[1]}" if c.batch[0] else str(c.batch[1])
    return f"{c.group}-{c.model}-T{c.T}-{b}"


def case_config(model):
    """The model config of a model id (no weights built)."""
    if model in HEAD_CASES:
        return head_config(model)
    name, ov = SHIPPED[model] if model in SHIPPED else _ROW[model][1:3]
    cfg, cleanup = _config(name, ov)
    cleanup()
    return cfg


def padmax_of(cfg):
    """The widest cache slice (dilation x (kernel_size - 1)) of a conv model."""
    bb = cfg["backbone"]
    if bb["type"] == "mdtc":
        return 2 ** (bb["stack_size"] - 1) * (bb["kernel_size"] - 1)
    return 2 ** (bb["num_layers"] - 1) * (bb.get("kernel_size", 8) - 1)


def conv_kernel(cfg):
    bb = cfg["backbone"]
    return "mdtc" if bb["type"] == "mdtc" else "dstcn" if bb.get("ds") else "tcn"


def batch_of(c, sms):
    if not isinstance(c.batch, str):
        return c.batch[0] * sms + c.batch[1]
    if c.batch == "linear":                       # B T just past 128 sms rows: some CTAs take two M tiles
        return kernel_constants()["linear_tc"] * sms // c.T + 11
    cfg = case_config(c.model)
    part = partition(conv_kernel(cfg), 1, c.T, padmax_of(cfg), sms)
    if c.batch == "tail":
        return sms * (2 * part["spt"] + 1)
    p = int(c.batch[1:])
    return sms * p * part["smax"] - sms // 2


def tensor_cores(c):
    """Whether the case's call must take a tensor-core kernel (uses_tensor_cores names it)."""
    return c.group in ("gru_tc", "conv", "dstcn", "linear") or (c.group == "head" and c.model != "tcn_global")


def classes(c, sms):
    """The partition classes one case reaches on `sms` SMs."""
    B = batch_of(c, sms)
    out = set()
    if c.group in ("gru_tc", "gru"):
        p = partition(c.group, B, c.T, 0, sms)
        if c.group == "gru_tc":
            out.add(f"gru_tc: {p['ms']} streams per tile" + ("" if p["partial"] else ", full tiles"))
            if p["partial"]:
                out.add("gru_tc: partial last tile")
        else:
            out.add(f"gru: {p['S']} streams per CTA")
        if p["tiles_per_cta"] >= 2:
            out.add(f"{c.group}: two tiles on one CTA")
        return out
    cfg = case_config(c.model)
    if c.group == "conv32":
        return {"conv fp32: T < 8"}
    kern = conv_kernel(cfg)
    head = c.group == "head"
    if head and kern != "mdtc":
        return {"tcn head: fp32 pool epilogue"}
    p = partition(kern, B, c.T, padmax_of(cfg), sms, head=head)
    if c.group == "linear":
        lp = partition("linear_tc", B, c.T, 0, sms)
        if lp["tiles_per_cta"] >= 2:
            out.add("linear_tc: two M tiles on one CTA")
        if lp["partial"]:
            out.add("linear_tc: partial M tile")
        if cfg["output_dim"] % 128:
            out.add("linear_tc: N tail")
        return out
    npass = max(len(ps) for ps in p["ctas"].values())
    if kern == "dstcn":
        return {f"dstcn: {min(npass, 3)}+ passes at chunk {p['chunk']}"} if npass >= 2 else set()
    name = "mdtc head" if head else kern
    out.add(f"{name}: {min(npass, 3)}{'+' if npass >= 3 else ''} pass{'es' if npass > 1 else ''}")
    all_passes = [q for ps in p["ctas"].values() for q in ps]
    if any(len(q["tiles"]) == 2 for q in all_passes):
        out.add(f"{name}: two tiles in a pass")
    if any(len(ps) >= 2 and len(ps[0]["tiles"]) == 2 and len(ps[-1]["tiles"]) == 1 for ps in p["ctas"].values()):
        out.add(f"{name}: last pass of one tile after a two-tile pass")
    if p["x_bound"] and any(len(q["tiles"]) and max(q["tiles"]) > 1 for q in all_passes):
        out.add(f"{name}: X columns bound the pass, several streams per tile")
    if 8 <= p["spt"] <= 14 and p["x_bound"]:
        out.add(f"{name}: 8..14 streams per tile (chunk 9..16), X-column bound")
    if p["spt"] == 1 and p["chunk"] > 64:
        out.add(f"{name}: one stream over both warpgroups")
    if p["smax"] == 1:
        out.add(f"{name}: one stream per pass")
    if kern == "mdtc" and not head:
        if any(q["ns"] > kernel_constants()["mdtc"]["NSLOT"] for q in all_passes):
            out.add("mdtc: more streams in a pass than landing slots")
        if any(s >= n_t > 1 for q in all_passes for s, n_t in zip(q["slots"], q["tiles"])):
            out.add("mdtc: a landing slot per stream, several streams per tile")
        if any(w == 1 for q in all_passes for w in q["wgs"]):
            out.add("mdtc: a tile on one warpgroup")
    if head:
        pool_spt = kernel_constants()["mdtc"]["POOL_SPT"]
        if p["spt"] == pool_spt and any(max(q["tiles"]) > 1 for q in all_passes):
            out.add("mdtc head: POOL_SPT streams per tile, several in a tile")
        if p["chunks"] >= 2 and max(p["ctas"]) > 2:
            out.add("mdtc head: pooled over several chunks, more than 2 streams per CTA")
    return out


REQUIRED = {
    "gru_tc: 16 streams per tile, full tiles", "gru_tc: 32 streams per tile", "gru_tc: 64 streams per tile",
    "gru_tc: partial last tile", "gru_tc: two tiles on one CTA",
    "gru: 2 streams per CTA", "gru: 4 streams per CTA", "gru: 8 streams per CTA", "gru: two tiles on one CTA",
    "linear_tc: two M tiles on one CTA", "linear_tc: partial M tile", "linear_tc: N tail",
    "mdtc: 1 pass", "mdtc: 2 passes", "mdtc: 3+ passes", "mdtc: two tiles in a pass",
    "mdtc: last pass of one tile after a two-tile pass", "mdtc: X columns bound the pass, several streams per tile",
    "mdtc: 8..14 streams per tile (chunk 9..16), X-column bound", "mdtc: one stream over both warpgroups",
    "mdtc: more streams in a pass than landing slots", "mdtc: a landing slot per stream, several streams per tile",
    "mdtc: a tile on one warpgroup",
    "tcn: 1 pass", "tcn: 2 passes", "tcn: 3+ passes", "tcn: two tiles in a pass",
    "tcn: last pass of one tile after a two-tile pass", "tcn: X columns bound the pass, several streams per tile",
    "tcn: 8..14 streams per tile (chunk 9..16), X-column bound", "tcn: one stream over both warpgroups",
    "tcn: one stream per pass",
    "dstcn: 2+ passes at chunk 8", "dstcn: 3+ passes at chunk 8", "dstcn: 3+ passes at chunk 60",
    "dstcn: 3+ passes at chunk 61", "dstcn: 3+ passes at chunk 120",
    "mdtc head: 1 pass", "mdtc head: 3+ passes", "mdtc head: two tiles in a pass",
    "mdtc head: POOL_SPT streams per tile, several in a tile",
    "mdtc head: pooled over several chunks, more than 2 streams per CTA",
    "tcn head: fp32 pool epilogue", "conv fp32: T < 8",
}


# ----------------------------------------------------------------------------------------------------------- CPU
def test_partition_constants_are_read_from_the_sources():
    K = kernel_constants()
    assert K["gru_tc"][1] > K["gru_tc"][3] > K["gru_tc"][4] and K["gru"][0] == 1
    assert K["mdtc"]["NSLOT_HEAD"] < K["mdtc"]["NSLOT"] and K["mdtc"]["POOL_SPT"] == K["mdtc"]["ROWS"] // 8
    assert K["dstcn"]["RPX"] >= 120 and K["linear_tc"] == 128


def test_partition_of_the_shipped_mdtc():
    """Hand-checked rows of the table: the shipped MDTC (padmax 32) at 1024 x 40 on 132 SMs runs its 8-stream CTAs
    as two passes of 3 + 1 streams (mdtc_tc.cu), at chunk 9 the X columns hold 12 streams."""
    p = partition("mdtc", 1024, 40, 32, 132)
    assert p["spt"] == 3 and p["smax"] == 6 and p["ctas"][8] == [
        dict(ns=4, tiles=[3, 1], slots=[3, 1], wgs=[2, 1]), dict(ns=4, tiles=[3, 1], slots=[3, 1], wgs=[2, 1])]
    p = partition("mdtc", 1, 9, 32, 132)
    assert p["spt"] == 14 and p["smax"] == 12 and p["x_bound"]
    assert partition("mdtc", 4 * 132 + 3, 300, 32, 132, head=True)["chunks"] == 3
    assert partition("tcn", 1, 56, 448, 132)["smax"] == 1


@pytest.mark.parametrize("sms", [132, 114])
def test_gpu_cases_reach_every_partition_class(sms):
    """The GPU shape list, mapped through the table, reaches every class in REQUIRED (H100 SXM: 132 SMs, PCIe: 114)."""
    reached = set()
    for c in CASES:
        reached |= classes(c, sms)
    missing = REQUIRED - reached
    assert not missing, sorted(missing)


def test_every_case_calls_one_chunk_height_or_the_head_chunks():
    """The conv cases call T frames in one chunk of T (the chunk height under test), except the 300-frame head calls
    and the two-chunk DS-TCN + linear_tc call."""
    for c in CASES:
        if c.group in ("conv", "dstcn"):
            cfg = case_config(c.model)
            assert partition(conv_kernel(cfg), 1, c.T, padmax_of(cfg), 132)["chunks"] == 1, case_id(c)


# ----------------------------------------------------------------------------------------------------------- GPU
DEV = "cuda:0"
_SLICE = 1 << 24            # oracle elements per slice of streams


@pytest.fixture(scope="module")
def models():
    cache = {}

    def get(model):
        if model not in cache:
            if model in HEAD_CASES:
                cfg, m = build_head_model(model, init_model)
            elif model in SHIPPED:
                cfg, m = build_config(*SHIPPED[model], init_model)
            else:
                cfg, m = build_row(model, init_model)
            # the float64 oracle: on the device for the conv models, on the host for the GRU (nn.GRU on the host)
            odev = "cpu" if cfg["backbone"]["type"] == "gru" else DEV
            sd = {k: (v.detach().to(odev, torch.float64) if v.dtype.is_floating_point else v.detach().to(odev))
                  for k, v in m.state_dict().items()}
            cache[model] = (cfg, m.to(DEV), sd, odev)
        return cache[model]
    yield get
    cache.clear()


def _compare(what, tc, cfg, sd, odev, x, cache, y, c):
    """Every stream of (y, c) against the float64 oracle, in slices of streams; asserts the sweep's gates."""
    B, T = x.shape[:2]
    gru = cfg["backbone"]["type"] == "gru"
    per = T * max(cfg["output_dim"], cfg["hidden_dim"]) + (cache[0].numel() if cache is not None and not gru else 0)
    step = max(1, _SLICE // per)
    ey = ec = my = mc = 0.0
    for s0 in range(0, B, step):
        s = slice(s0, min(B, s0 + step))
        cs = None if cache is None else (cache[:, s] if gru else cache[s]).to(odev, torch.float64)
        y_ref, c_ref = HO.kws_forward(sd, cfg, x[s].to(odev, torch.float64), cs)
        ys, cs_out = y[s], (c[:, s] if gru else c[s])
        ey = max(ey, float((ys.to(odev, torch.float64) - y_ref).abs().max()))
        ec = max(ec, float((cs_out.to(odev, torch.float64) - c_ref).abs().max()))
        my, mc = max(my, float(y_ref.abs().max())), max(mc, float(c_ref.abs().max()))
    gy, gc = _gate(tc, torch.tensor(my)), _gate(tc, torch.tensor(mc))
    print(f"{what} {'tensor-core' if tc else 'fp32'}: out {ey:.2e} (gate {gy:.1e}), cache {ec:.2e} (gate {gc:.1e})")
    assert ey <= gy and ec <= gc, (what, ey, gy, ec, gc)


def _precision(c):
    return "tensor" if c.group == "gru_tc" else "fp32" if c.group == "gru" else "auto"


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_gpu_every_stream_matches_float64_oracle(c, models):
    """Every stream's output and returned cache against the float64 oracle, from a random cache and from none; the
    call takes the kernel the case is for."""
    cfg, m, sd, odev = models(c.model)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = batch_of(c, sms)
    x, cache = inputs(cfg, B, c.T, seed=7 * B + c.T)
    tc = tensor_cores(c)
    xd = x.to(DEV)
    try:
        m.precision = _precision(c)
        for name, cin in (("random cache", cache), ("no cache", None)):
            y, cout = m(xd) if cin is None else m(xd, cin.to(DEV))
            assert m.uses_tensor_cores(c.T, B) == tc, (case_id(c), B)
            _compare(f"{case_id(c)} B={B} {name}", tc, cfg, sd, odev, x, cin, y, cout)
    finally:
        m.precision = "auto"


@pytest.mark.gpu
@pytest.mark.parametrize("b", _GRU_TC_B, ids=lambda b: f"{b[0]}sms+{b[1]}")
@pytest.mark.parametrize("model", ["gru", "gru_1l_i40", "gru_i13"])
def test_gpu_gru_tc_carried_calls_equal_one_call(model, b, models):
    """Tensor-core GRU: 1 frame, then 2 with the cache carried, equal one call of 3 frames bit for bit (the state
    crosses the call in fp32 exactly as it crosses a step)."""
    cfg, m, _, _ = models(model)
    B = b[0] * torch.cuda.get_device_properties(0).multi_processor_count + b[1]
    x, cache = inputs(cfg, B, 3, seed=31 + B)
    xd, cd = x.to(DEV), cache.to(DEV)
    try:
        m.precision = "tensor"
        y, c = m(xd, cd)
        y1, c1 = m(xd[:, :1].contiguous(), cd)
        y2, c2 = m(xd[:, 1:].contiguous(), c1)
    finally:
        m.precision = "auto"
    assert torch.equal(torch.cat([y1, y2], 1), y) and torch.equal(c2, c), (model, B)


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["gru", "gru_1l_i40", "gru_i13"])
def test_gpu_gru_tc_stream_permutation_with_two_tiles_per_cta(model, models):
    """64 sms + 37 streams (two tiles on some CTAs, a partial last tile): permuting the streams permutes the outputs
    and caches bit for bit."""
    cfg, m, _, _ = models(model)
    B = 64 * torch.cuda.get_device_properties(0).multi_processor_count + 37
    x, cache = inputs(cfg, B, 3, seed=5)
    xd, cd = x.to(DEV), cache.to(DEV)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(1)).to(DEV)
    try:
        m.precision = "tensor"
        y, c = m(xd, cd)
        yp, cp = m(xd[perm].contiguous(), cd[:, perm].contiguous())
    finally:
        m.precision = "auto"
    assert torch.equal(yp, y[perm]) and torch.equal(cp, c[:, perm]), model
