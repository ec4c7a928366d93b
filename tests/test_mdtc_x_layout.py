"""CPU check of the shared-memory layout of the MDTC tensor-core kernel's residual stream X (wekws_b200/csrc/mdtc_tc.cu).

X holds 64 fp32 channels per frame column.  The kernel pads each column to 272 bytes (one spare 16-byte chunk), so
chunk m of column col sits in bank group (col + m) mod 8 and the chunk offset 16 m is an immediate of the load; the
layout it replaced kept 256-byte columns and XOR-swizzled the chunk index with (col & 7).  For every access pattern the
kernel makes of X -- the wgmma-fragment rows (first-Linear store, depthwise taps, residual load and store), the
cache-slice loads, the loaders' transposes and zero fill, and the head variant's pooling -- and for every slice width
and chunk length the kernel accepts, the test counts the shared-memory wavefronts of each warp-wide access under both
layouts and requires the padded one never to need more.  The lane -> (column, channel) maps restate the kernel's index
formulas; the address formula is read from the source, so the test fails if the layout changes without this restatement.
"""
import os
import re

import numpy as np

from tests.conftest import ROOT

SRC = open(os.path.join(ROOT, "wekws_b200", "csrc", "mdtc_tc.cu")).read()
XCOLS = 504
LANE = np.arange(32)


def padded(col, ch):
    """x_addr(0, col, ch) as the kernel defines it."""
    return col * 272 + 16 * (ch >> 3) + 128 * ((ch >> 2) & 1) + 4 * (ch & 3)


def swizzled(col, ch):
    """The previous layout: address(col, 8m + 4h + u) = ((col << 8) | ((col & 7) << 4)) ^ (m << 4) + 128 h + 4 u."""
    return (((col << 8) | ((col & 7) << 4)) ^ ((ch >> 3) << 4)) + 128 * ((ch >> 2) & 1) + 4 * (ch & 3)


def test_source_uses_the_restated_layout():
    assert re.search(r"constexpr int X_COL = 272;", SRC), "X column stride changed: update this test"
    assert re.search(r"return xs \+ \(uint32_t\)col \* X_COL \+ 16u \* \(uint32_t\)\(ch >> 3\) \+ "
                     r"128u \* \(uint32_t\)\(\(ch >> 2\) & 1\) \+ 4u \* \(uint32_t\)\(ch & 3\);", SRC), \
        "x_addr changed: update this test"
    assert re.search(rf"constexpr int XCOLS = {XCOLS};", SRC)
    # every X access goes through x_addr (the fragment rows through t_own / tj, formed by it): no other column stride
    assert not re.search(r"<< 8\)|col & 7|cc & 7", SRC)


def wavefronts(addr, width):
    """Wavefronts of warp-wide accesses: addr (n, 32) byte addresses (-1: inactive lane), each lane accessing `width`
    bytes.  A wavefront serves one distinct 4-byte word per bank, so the count is the largest number of distinct words
    any bank is asked for (lanes asking for the same word share it)."""
    n = addr.shape[0]
    k = width // 4
    words = (addr[:, :, None] // 4 + np.arange(k)).reshape(n, -1)
    words = np.where(np.repeat(addr >= 0, k, axis=1), words, -1)
    words.sort(axis=1)
    first = np.ones_like(words, bool)
    first[:, 1:] = words[:, 1:] != words[:, :-1]
    first &= words >= 0
    idx = np.nonzero(first)
    per_bank = np.zeros((n, 32), np.int64)
    np.add.at(per_bank, (idx[0], words[idx] % 32), 1)
    return per_bank.max(1)


def compare(old, new, width):
    """(old, new) wavefront counts of the same accesses; a shift by a multiple of 128 bytes keeps every bank, so the
    accesses are normalised and deduplicated first."""
    def norm(a):
        lo = np.where(a >= 0, a, np.iinfo(a.dtype).max).min(1, keepdims=True)
        return np.where(a >= 0, a - 128 * (lo // 128), -1)
    pairs = np.unique(np.concatenate([norm(old), norm(new)], 1), axis=0)
    return wavefronts(pairs[:, :32], width), wavefronts(pairs[:, 32:], width)


def tiles(T, ns):
    spt = 128 // T
    return [(g, min(spt, ns - g * spt)) for g in range(2) if ns - g * spt > 0]


def patterns(padr, T, ns):
    """Every warp-wide access the kernel makes of X at this shape: name -> (width, old addresses, new addresses)."""
    spt, Lw = 128 // T, padr + T
    pads = [p for p in (4, 8, 16, 32) if p <= padr]
    acc = {}

    def add(name, width, col, ch, old=None):
        col, ch = np.broadcast_arrays(col, ch)
        col, ch = col.reshape(-1, 32), ch.reshape(-1, 32)
        new = np.where(col >= 0, padded(col, ch), -1)
        old = np.where(col >= 0, swizzled(col, ch), -1) if old is None else old.reshape(-1, 32)
        w, o, n = acc.get(name, (width, [], []))
        acc[name] = (w, o + [old], n + [new])

    # wgmma-fragment rows: warp wq of tile g holds rows r0 + 8 h, r0 = 64 (wq >> 2) + 16 (wq & 3) + lane / 4, channel
    # pair 8 m + 2 (lane & 3); a dead row aliases its tile's first frame.  The own column (first-Linear store, residual
    # load and store) and the depthwise taps col - pad + j d (K = 2, 3, 5 taps over a power-of-two slice)
    offs = sorted({-pad + j * d for pad in pads for d in {pad, pad // 2, pad // 4} - {0} for j in range(pad // d + 1)})
    cols = []
    for g, nst in tiles(T, ns):
        for wq in range(8):
            for h in range(2):
                row = 64 * (wq >> 2) + 16 * (wq & 3) + LANE // 4 + 8 * h
                live = row < nst * T
                cols.append((g * spt + np.where(live, row // T, 0)) * Lw + padr + np.where(live, row % T, 0))
    cols = np.array(cols)[:, None, None, :] + np.array(offs)[None, :, None, None]
    add("fragment", 8, cols, 8 * np.arange(8)[None, None, :, None] + 2 * (LANE & 3))

    for pad in pads:
        # cache-slice loads (LDS.128): 8 lanes per cache row of jpl columns, quads of channels cq
        jpl = min(pad, 32)
        lgj = jpl.bit_length() - 1
        qstep, per = 32 >> lgj, 16 >> (5 - lgj)
        j, qs = LANE & (jpl - 1), LANE >> lgj
        lgg = (pad >> 2).bit_length() - 1
        pi = 16 << lgg
        for g, nst in tiles(T, ns):
            # (the swizzled layout took quad q; the padded one takes q with its chunk index q >> 1 rotated by a bit)
            it = np.arange(nst * per)[:, None]
            s2 = it // per
            col, q = (g * spt + s2) * Lw + padr + T - pad + j, (it - s2 * per) * qstep + qs
            mq = q >> 1
            add("cache-slice load", 16, col, 4 * (2 * (((mq << 1) | (mq >> 2)) & 7) + (q & 1)),
                old=swizzled(*np.broadcast_arrays(col, 4 * q)))
            # loader transposes (STS.128), the flat loop over the tile's streams: item -> stream m, channel quad cq,
            # column group jg; four stores, one per column of the group
            it = np.arange(0, nst * pi, 32)[:, None] + LANE
            m, r = it >> (4 + lgg), it & (pi - 1)
            cq, jg = r >> lgg, r & ((1 << lgg) - 1)
            for e in range(4):
                add("loader transpose", 16, np.where(it < nst * pi, (g * spt + m) * Lw + padr - pad + 4 * jg + e, -1),
                    4 * cq)
            # no incoming cache: zero fill of the slice's columns, 16 bytes per lane (the old layout wrote them as one
            # contiguous range)
            e = np.arange(0, pad * 16, 32)[:, None] + LANE
            colb = g * spt * Lw + padr - pad
            add("loader zero fill", 16, colb + (e >> 4), 4 * (e & 15), old=colb * 256 + 16 * e)
    # head pooling (LDS.32, head variant: spt <= 16): warp wq, lane = 8 q + channel, frames t = q, q + 4, ...
    if spt <= 16:
        for g, nst in tiles(T, ns):
            t = np.arange(0, T, 4)[:, None] + (LANE >> 3)
            for wq in range(8):
                for s2 in range(nst):
                    add("head pooling", 4, np.where(t < T, (g * spt + s2) * Lw + padr + t, -1), 8 * wq + (LANE & 7))
    return {k: (w, np.concatenate(o), np.concatenate(n)) for k, (w, o, n) in acc.items()}


def shapes():
    """(padr, T, ns): every slice width and chunk length the kernel accepts (tc_eligible: power-of-two slices of 4..32
    columns, padr = the widest; mdtc_tc_launch: T <= 128, spt = 128 / T streams per tile, two tiles per pass, padr + T
    columns per stream, XCOLS columns in all), each with one stream, two, and a full pass."""
    for padr in (4, 8, 16, 32):
        for T in range(1, 129):
            smax = min(2 * (128 // T), XCOLS // (padr + T))
            for ns in sorted({1, min(2, smax), smax}):
                yield padr, T, ns


def test_padded_layout_never_needs_more_wavefronts_than_the_swizzle():
    worse, seen = [], set()
    for padr, T, ns in shapes():
        for name, (width, old, new) in patterns(padr, T, ns).items():
            o, n = compare(old, new, width)
            seen.add(name)
            if (n > o).any():
                worse.append((name, padr, T, ns, int(n.max()), int(o.max())))
    assert seen == {"fragment", "cache-slice load", "loader transpose", "loader zero fill", "head pooling"}
    assert not worse, f"padded layout needs more wavefronts than the swizzle: {worse[:10]}"


def test_flagship_accesses_take_the_minimum_wavefronts():
    """At the flagship shape (cache slices of 4 to 32 columns, T = 40, a pass of 3 + 1 streams) every fragment access
    takes the two wavefronts of a 256-byte warp access, and every cache-slice load the four of a 512-byte one (the
    swizzled layout needed eight for the 4-column slices)."""
    acc = patterns(32, 40, 4)
    for name, minimum in (("fragment", 2), ("cache-slice load", 4)):
        width, old, new = acc[name]
        assert compare(old, new, width)[1].max() == minimum, name
