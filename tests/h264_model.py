"""A numpy model of the encoder's operations, written from ITU-T H.264 (8.3, 8.4.2.2, 8.5) and DESIGN.md §5.2 (the intra decision) /
§5.3 (wide-range motion included) / §5.4 / §5.7, in int64.
It shares no code with oracle/ or selkies_b200/.  Planes are 2-D uint8 arrays of the coded size (chroma: one array per
component); coordinates are in samples of the plane.  The 4x4 operations also take a stack of blocks (..., 4, 4)."""
from __future__ import annotations

import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

from tests.h264_syntax import BLK_IDX, BLK_XY, CDC_TOKEN, CDC_TOTAL_ZEROS, COEFF_TOKEN, RUN_BEFORE, TOTAL_ZEROS, ZIGZAG_XY

# 8.5.9 / §5.4: quantisation multipliers MF and dequantisation scales v per qp % 6 for the position classes
# (both coordinates even, both odd, otherwise)
MF = [(13107, 5243, 8066), (11916, 4660, 7490), (10082, 4194, 6554), (9362, 3647, 5825), (8192, 3355, 5243), (7282, 2893, 4559)]
V = [(10, 16, 13), (11, 18, 14), (13, 20, 16), (14, 23, 18), (16, 25, 20), (18, 29, 23)]
# Table 8-15: QPc from qPI
QPC = list(range(30)) + [29, 30, 31, 32, 32, 33, 34, 34, 35, 35, 36, 36, 37, 37, 37, 38, 38, 38, 39, 39, 39, 39]
# §5.3: motion-search Lagrangian per QP
LAMBDA = [1] * 20 + [2, 2, 2, 2, 3, 3, 3, 4, 4, 4, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 23, 25, 29, 32, 36, 40, 45, 51, 57]
EARLY_SAD_PER_LAMBDA = 96
REFINE_MAX_SAD = 8192
FRAC_PENALTY_BITS = 4


def pos_class(x, y):
    return 0 if x % 2 == 0 and y % 2 == 0 else 1 if x % 2 == 1 and y % 2 == 1 else 2


CLASS = np.array([[pos_class(x, y) for x in range(4)] for y in range(4)])


def mf_of(qp):
    return np.array(MF[qp % 6], np.int64)[CLASS]


def v_of(qp):
    return np.array(V[qp % 6], np.int64)[CLASS]


def clip1(a):
    return np.clip(a, 0, 255)


# ------------------------------------------------------------------------------------------------ transforms (8.5)
CF = np.array([[1, 1, 1, 1], [2, 1, -1, -2], [1, -1, -1, 1], [1, -2, 2, -1]], np.int64)
H4 = np.array([[1, 1, 1, 1], [1, 1, -1, -1], [1, -1, -1, 1], [1, -1, 1, -1]], np.int64)
H2 = np.array([[1, 1], [1, -1]], np.int64)


def forward4x4(x):
    """The forward core transform W = Cf X Cf^T of a 4x4 residual."""
    return CF @ np.asarray(x, np.int64) @ CF.T


def quant(w, mf, f, qbits):
    """§5.4: |l| = (|w|·MF + f) >> qbits, the sign of w, |l| <= 2047."""
    w = np.asarray(w, np.int64)
    return np.sign(w) * np.minimum((np.abs(w) * mf + f) >> qbits, 2047)


def dead_zone(qbits, intra):
    return (1 << qbits) // (3 if intra else 6)


def inverse4x4(d):
    """8.5.12.2: rows, then columns, then (x + 32) >> 6 (of each 4x4 block of a stack)."""
    d = np.asarray(d, np.int64)

    def one(v):                                          # v[..., 0..3]
        e0, e1 = v[..., 0] + v[..., 2], v[..., 0] - v[..., 2]
        e2, e3 = (v[..., 1] >> 1) - v[..., 3], v[..., 1] + (v[..., 3] >> 1)
        return np.stack([e0 + e3, e1 + e2, e1 - e2, e0 - e3], axis=-1)
    f = one(d)                                           # each row
    h = np.swapaxes(one(np.swapaxes(f, -1, -2)), -1, -2)  # each column
    return (h + 32) >> 6


def dequant4x4(c, qp, skip_dc=False):
    """8.5.12.1 with flat weights (LevelScale4x4 = 16 · v)."""
    ls = 16 * v_of(qp)
    c = np.asarray(c, np.int64)
    d = (c * ls) << (qp // 6 - 4) if qp >= 24 else (c * ls + (1 << (3 - qp // 6))) >> (4 - qp // 6)
    if skip_dc:
        d[..., 0, 0] = 0
    return d


def luma_dc_dequant(c, qp):
    """8.5.10: inverse Hadamard of the Intra16x16 DC levels (4x4 raster of blocks) and their scaling."""
    f = H4 @ np.asarray(c, np.int64) @ H4
    ls = 16 * V[qp % 6][0]
    return (f * ls) << (qp // 6 - 6) if qp >= 36 else (f * ls + (1 << (5 - qp // 6))) >> (6 - qp // 6)


def chroma_dc_dequant(c, qpc):
    """8.5.11.1-2: inverse 2x2 Hadamard of the chroma DC levels (2x2 raster) and their scaling."""
    f = H2 @ np.asarray(c, np.int64) @ H2
    return ((f * 16 * V[qpc % 6][0]) << (qpc // 6)) >> 5


def quant_block(res, qp, intra, with_dc=True):
    """Forward transform and quantisation of one 4x4 residual; returns (raster levels, raw W).  The DC level is 0 when the
    caller codes the DC separately."""
    w = forward4x4(res)
    qbits = 15 + qp // 6
    lv = quant(w, mf_of(qp), dead_zone(qbits, intra), qbits)
    if not with_dc:
        lv[..., 0, 0] = 0
    return lv, w


def i16_dc_levels(w_dc, qp):
    """§5.4 Intra16x16 DC path: Hadamard of the 16 forward DCs (4x4 raster of blocks), (acc + 1) >> 1, 2f and qbits + 1."""
    acc = H4 @ np.asarray(w_dc, np.int64) @ H4
    qbits = 15 + qp // 6
    return quant((acc + 1) >> 1, MF[qp % 6][0], 2 * dead_zone(qbits, True), qbits + 1)


def chroma_dc_levels(w_dc, qpc, intra):
    """§5.4 chroma DC path: 2x2 Hadamard of the four forward DCs, 2f and qbits + 1."""
    acc = H2 @ np.asarray(w_dc, np.int64) @ H2
    qbits = 15 + qpc // 6
    return quant(acc, MF[qpc % 6][0], 2 * dead_zone(qbits, intra), qbits + 1)


def decimation_score(levels_scan):
    """§5.4: 9 if any |level| > 1, else the sum over the ±1 levels of {3,2,2,1,1,1,0...}[zeros just below it in scan order]."""
    if np.any(np.abs(levels_scan) > 1):
        return 9
    table = [3, 2, 2, 1, 1, 1]
    score, zeros = 0, 0
    for v in levels_scan:
        if v == 0:
            zeros += 1
            continue
        score += table[zeros] if zeros < 6 else 0
        zeros = 0
    return score


def decimate_levels(luma_scan):
    """§5.4 inter-luma decimation of (16 blkIdx, 16 scan) levels: an 8x8 quadrant scoring < 4 is zeroed, all of it when the
    macroblock scores < 6."""
    out = luma_scan.copy()
    s = [decimation_score(luma_scan[b]) for b in range(16)]
    quad = [sum(s[4 * q: 4 * q + 4]) for q in range(4)]
    for b in range(16):
        if quad[b >> 2] < 4 or sum(s) < 6:
            out[b] = 0
    return out


_ZX, _ZY = (np.array(c) for c in zip(*ZIGZAG_XY))


def raster_to_scan(r):
    """The 16 levels of a 4x4 raster block (or of each block of a stack) in zig-zag scan order."""
    return np.asarray(r, np.int64)[..., _ZY, _ZX]


# ------------------------------------------------------------------------------------------------ the I_PCM rule (§5.7)
def _lengths(table):
    return {v: len(code) for code, v in table.items()}


_TOKEN, _CDC_TOKEN = [_lengths(t) for t in COEFF_TOKEN], _lengths(CDC_TOKEN)
_TZ, _CDC_TZ, _RUN = [_lengths(t) for t in TOTAL_ZEROS], [_lengths(t) for t in CDC_TOTAL_ZEROS], [_lengths(t) for t in RUN_BEFORE]
HEADER_BITS = 48                 # §5.7: the header budget of a macroblock; 96 for Intra4x4 (its prediction modes)
WM_MVD_BITS = 48                 # §5.3: 48 more for a P macroblock of a wide-motion picture (two mvd of up to ±2046)


def cavlc_bits(scan, chroma_dc=False):
    """9.2: the length of residual_block_cavlc() for the levels `scan` (scan order, maxNumCoeff = len(scan)), with the longest
    coeff_token of the four nC tables (§5.7: a size taken before the neighbours' counts are known), the chroma DC table for
    chroma_dc."""
    nz = [k for k, v in enumerate(scan) if v]
    total = len(nz)
    lv = [int(scan[k]) for k in reversed(nz)]            # highest frequency first
    t1 = 0
    while t1 < min(3, total) and abs(lv[t1]) == 1:
        t1 += 1
    bits = _CDC_TOKEN[(total, t1)] if chroma_dc else max(t.get((total, t1), 0) for t in _TOKEN)
    if not total:
        return bits
    suffix_len = 1 if total > 10 and t1 < 3 else 0
    for i, v in enumerate(lv):
        if i < t1:
            bits += 1                                    # trailing_ones_sign_flag
            continue
        code = 2 * v - 2 if v > 0 else -2 * v - 1        # 9.2.2.1 levelCode
        if i == t1 and t1 < 3:
            code -= 2
        if suffix_len == 0:
            bits += code + 1 if code < 14 else 19 if code < 30 else 28      # level_prefix 14 + 4 suffix bits; 15 + 12
        else:
            bits += (code >> suffix_len) + 1 + suffix_len if code < 15 << suffix_len else 28
        if suffix_len == 0:
            suffix_len = 1
        if abs(v) > 3 << (suffix_len - 1) and suffix_len < 6:
            suffix_len += 1
    zeros = nz[-1] + 1 - total
    if total < len(scan):
        bits += (_CDC_TZ if chroma_dc else _TZ)[total - 1][zeros]
    for i in range(total - 1):                           # run_before, highest frequency first, while zeros are left
        if zeros <= 0:
            break
        run = nz[-1 - i] - nz[-2 - i] - 1
        bits += _RUN[min(zeros, 7) - 1][run]
        zeros -= run
    return bits


def header_budget(m, wide=False):
    """§5.7 / §5.3 / §5.13: the bits budgeted for everything of macroblock `m` before its residual — mb_type, ref_idx_l0 (one bit in a
    picture with two references), mvd, coded_block_pattern and mb_qp_delta: 48, 96 for Intra4x4 (its prediction modes), 48 more for
    a P macroblock of a wide-motion picture."""
    return HEADER_BITS + (HEADER_BITS if m.kind == "I_NxN" else 0) + (WM_MVD_BITS if wide and not m.intra else 0)


def mb_size_estimate(m, wide=False):
    """§5.7 / §5.3: the size the encoders give a parsed macroblock `m` (not I_PCM, not P_Skip) when they decide whether to send it
    raw: its coded blocks by cavlc_bits, plus header_budget().  Above 3200 the macroblock is I_PCM."""
    bits = header_budget(m, wide)
    i16 = m.kind == "I_16x16"
    if i16:
        bits += cavlc_bits(m.luma_dc)
    for blk in range(16):
        if m.cbp >> (blk >> 2) & 1:
            bits += cavlc_bits(m.luma[blk][1:] if i16 else m.luma[blk])
    if m.cbp >> 4:
        bits += sum(cavlc_bits(m.chroma_dc[c], chroma_dc=True) for c in range(2))
    if m.cbp >> 4 & 2:
        bits += sum(cavlc_bits(m.chroma_ac[c][blk][1:]) for c in range(2) for blk in range(4))
    return bits


# ------------------------------------------------------------------------------------------------ intra prediction (8.3)
class Avail:
    """Neighbour availability of one macroblock: left A, top B, top-right C, top-left D (6.4.11.1)."""

    def __init__(self, a, b, c, d):
        self.a, self.b, self.c, self.d = a, b, c, d


def intra4x4_pred(mode, P):
    """8.3.1.2.1-9: P(x, y) for x, y in -1..7 gives p[x, y] (None when not available): one sample, or an array of one sample per
    block of a stack.  Returns the 4x4 raster (the stack of them, (..., 4, 4)); ValueError when the mode reads a sample that is not
    available."""
    vals = []
    for y in range(4):
        for x in range(4):
            if mode == 0:
                v = P(x, -1)
            elif mode == 1:
                v = P(-1, y)
            elif mode == 2:
                top = [P(i, -1) for i in range(4)]
                left = [P(-1, i) for i in range(4)]
                has_top, has_left = all(t is not None for t in top), all(t is not None for t in left)
                if has_top and has_left:
                    v = (sum(top) + sum(left) + 4) >> 3
                elif has_left:
                    v = (sum(left) + 2) >> 2
                elif has_top:
                    v = (sum(top) + 2) >> 2
                else:
                    v = 128
            elif mode == 3:
                v = (P(6, -1) + 3 * P(7, -1) + 2) >> 2 if x == 3 and y == 3 else \
                    (P(x + y, -1) + 2 * P(x + y + 1, -1) + P(x + y + 2, -1) + 2) >> 2
            elif mode == 4:
                if x > y:
                    v = (P(x - y - 2, -1) + 2 * P(x - y - 1, -1) + P(x - y, -1) + 2) >> 2
                elif x < y:
                    v = (P(-1, y - x - 2) + 2 * P(-1, y - x - 1) + P(-1, y - x) + 2) >> 2
                else:
                    v = (P(0, -1) + 2 * P(-1, -1) + P(-1, 0) + 2) >> 2
            elif mode == 5:
                z = 2 * x - y
                if z >= 0 and z % 2 == 0:
                    v = (P(x - (y >> 1) - 1, -1) + P(x - (y >> 1), -1) + 1) >> 1
                elif z >= 0:
                    v = (P(x - (y >> 1) - 2, -1) + 2 * P(x - (y >> 1) - 1, -1) + P(x - (y >> 1), -1) + 2) >> 2
                elif z == -1:
                    v = (P(-1, 0) + 2 * P(-1, -1) + P(0, -1) + 2) >> 2
                else:
                    v = (P(-1, y - 1) + 2 * P(-1, y - 2) + P(-1, y - 3) + 2) >> 2
            elif mode == 6:
                z = 2 * y - x
                if z >= 0 and z % 2 == 0:
                    v = (P(-1, y - (x >> 1) - 1) + P(-1, y - (x >> 1)) + 1) >> 1
                elif z >= 0:
                    v = (P(-1, y - (x >> 1) - 2) + 2 * P(-1, y - (x >> 1) - 1) + P(-1, y - (x >> 1)) + 2) >> 2
                elif z == -1:
                    v = (P(-1, 0) + 2 * P(-1, -1) + P(0, -1) + 2) >> 2
                else:
                    v = (P(x - 1, -1) + 2 * P(x - 2, -1) + P(x - 3, -1) + 2) >> 2
            elif mode == 7:
                if y % 2 == 0:
                    v = (P(x + (y >> 1), -1) + P(x + (y >> 1) + 1, -1) + 1) >> 1
                else:
                    v = (P(x + (y >> 1), -1) + 2 * P(x + (y >> 1) + 1, -1) + P(x + (y >> 1) + 2, -1) + 2) >> 2
            else:
                z = x + 2 * y
                if z > 5:
                    v = P(-1, 3)
                elif z == 5:
                    v = (P(-1, 2) + 3 * P(-1, 3) + 2) >> 2
                elif z % 2 == 0:
                    v = (P(-1, y + (x >> 1)) + P(-1, y + (x >> 1) + 1) + 1) >> 1
                else:
                    v = (P(-1, y + (x >> 1)) + 2 * P(-1, y + (x >> 1) + 1) + P(-1, y + (x >> 1) + 2) + 2) >> 2
            if v is None:
                raise ValueError(f"Intra4x4 mode {mode} uses an unavailable sample")
            vals.append(np.asarray(v, np.int64))
    out = np.stack(vals).reshape(4, 4, *vals[0].shape)
    return np.moveaxis(out, (0, 1), (-2, -1))


def intra4x4_accessor(get, blk, av: Avail):
    """p[x, y] accessor for luma block blk of a macroblock with the availability rules of 6.4.11.4 and the top-right substitution
    of 8.3.1.2; get(nx, ny) reads the sample at offset (nx, ny) from the macroblock's top-left corner of the picture being
    decoded."""
    bx, by = BLK_XY[blk]

    def avail(nx, ny):                                   # (nx, ny): sample offset relative to the macroblock
        if nx < 0 and ny < 0:
            return av.d if (bx == 0 and by == 0) else (av.a if bx == 0 else av.b if by == 0 else True)
        if nx < 0:
            return av.a if bx == 0 else True
        if ny < 0:
            if nx >= 16:
                return av.c
            return av.b
        if nx >= 16:
            return False
        return BLK_IDX[(nx // 4, ny // 4)] < blk         # inside the macroblock: decoded earlier

    have_c = avail(bx * 4 + 4, by * 4 - 1)
    have_b = avail(bx * 4, by * 4 - 1)

    def P(x, y):
        if x > 3 and y == -1 and not have_c:
            if not have_b:
                return None
            x = 3
        if not avail(bx * 4 + x, by * 4 + y):
            return None
        return get(bx * 4 + x, by * 4 + y)
    return P


def intra4x4_neighbours(rec, mbx, mby, blk, av: Avail):
    """intra4x4_accessor for luma block blk of macroblock (mbx, mby) reading the picture `rec` being decoded."""
    x0, y0 = mbx * 16, mby * 16
    return intra4x4_accessor(lambda nx, ny: int(rec[y0 + ny, x0 + nx]), blk, av)


def intra16_pred(mode, top, left, tl):
    """8.3.3: top / left are 16-sample arrays or None, tl the corner sample or None."""
    if mode == 0:
        return np.tile(np.asarray(top, np.int64), (16, 1))
    if mode == 1:
        return np.tile(np.asarray(left, np.int64)[:, None], (1, 16))
    if mode == 2:
        if top is not None and left is not None:
            v = (int(np.sum(top)) + int(np.sum(left)) + 16) >> 5
        elif left is not None:
            v = (int(np.sum(left)) + 8) >> 4
        elif top is not None:
            v = (int(np.sum(top)) + 8) >> 4
        else:
            v = 128
        return np.full((16, 16), v, np.int64)
    t = np.concatenate([[tl], top]).astype(np.int64)     # t[i + 1] = p[i, -1]
    l_ = np.concatenate([[tl], left]).astype(np.int64)
    H = sum((i + 1) * (t[8 + i + 1] - t[6 - i + 1]) for i in range(8))
    Vv = sum((i + 1) * (l_[8 + i + 1] - l_[6 - i + 1]) for i in range(8))
    a, b, c = 16 * (int(left[15]) + int(top[15])), (5 * H + 32) >> 6, (5 * Vv + 32) >> 6
    y, x = np.mgrid[0:16, 0:16]
    return clip1((a + b * (x - 7) + c * (y - 7) + 16) >> 5)


def chroma_pred(mode, top, left, tl):
    """8.3.4 for 4:2:0 (8x8 per component)."""
    if mode == 2:
        return np.tile(np.asarray(top, np.int64), (8, 1))
    if mode == 1:
        return np.tile(np.asarray(left, np.int64)[:, None], (1, 8))
    if mode == 0:
        out = np.zeros((8, 8), np.int64)
        for yo in (0, 4):
            for xo in (0, 4):
                st = None if top is None else int(np.sum(top[xo:xo + 4]))
                sl = None if left is None else int(np.sum(left[yo:yo + 4]))
                if (xo, yo) in ((0, 0), (4, 4)):
                    v = (st + sl + 4) >> 3 if st is not None and sl is not None else \
                        (sl + 2) >> 2 if sl is not None else (st + 2) >> 2 if st is not None else 128
                elif yo == 0:
                    v = (st + 2) >> 2 if st is not None else (sl + 2) >> 2 if sl is not None else 128
                else:
                    v = (sl + 2) >> 2 if sl is not None else (st + 2) >> 2 if st is not None else 128
                out[yo:yo + 4, xo:xo + 4] = v
        return out
    t = np.concatenate([[tl], top]).astype(np.int64)
    l_ = np.concatenate([[tl], left]).astype(np.int64)
    H = sum((i + 1) * (t[4 + i + 1] - t[2 - i + 1]) for i in range(4))
    Vv = sum((i + 1) * (l_[4 + i + 1] - l_[2 - i + 1]) for i in range(4))
    a, b, c = 16 * (int(left[7]) + int(top[7])), (34 * H + 32) >> 6, (34 * Vv + 32) >> 6
    y, x = np.mgrid[0:8, 0:8]
    return clip1((a + b * (x - 3) + c * (y - 3) + 16) >> 5)


def mb_edges(plane, x0, y0, n, av: Avail):
    """Top / left / top-left neighbours of the n x n block at (x0, y0) of a decoded plane."""
    top = plane[y0 - 1, x0:x0 + n].astype(np.int64) if av.b else None
    left = plane[y0:y0 + n, x0 - 1].astype(np.int64) if av.a else None
    tl = int(plane[y0 - 1, x0 - 1]) if av.d else None
    return top, left, tl


# ------------------------------------------------------------------------------------------------ inter prediction (8.4.2.2)
TAP = np.array([1, -5, 20, 20, -5, 1], np.int64)


def luma_inter(ref, x0, y0, mv, n=16, rows=None):
    """8.4.2.2.1: the n x n luma prediction at (x0, y0) for quarter-sample vector mv, reference coordinates clamped to the
    plane (rows = (first, last) row for a band-clamped reference)."""
    return luma_planes(ref, x0 + (mv[0] >> 2), y0 + (mv[1] >> 2), n, rows)[(mv[0] & 3, mv[1] & 3)]


def luma_planes(ref, xi, yi, n=16, rows=None):
    """8.4.2.2.1: {(xFrac, yFrac): the n x n luma prediction whose full-sample part is the position (xi, yi)}, all sixteen from one
    set of half-sample planes."""
    h, w = ref.shape
    r0, r1 = rows if rows is not None else (0, h - 1)
    ys = np.clip(np.arange(yi - 2, yi + n + 4), r0, r1)
    xs = np.clip(np.arange(xi - 2, xi + n + 4), 0, w - 1)
    W = ref[np.ix_(ys, xs)].astype(np.int64)             # W[r + 2, c + 2] = sample (xi + c, yi + r)
    b1 = sum(TAP[k] * W[:, k:k + n] for k in range(6))    # (n + 6, n): half sample right of (c, r), rows r = -2 .. n + 3
    h1 = sum(TAP[k] * W[k:k + n, :] for k in range(6))    # (n, n + 6): half sample below (c, r), columns c = -2 .. n + 3
    j1 = sum(TAP[k] * b1[k:k + n, :] for k in range(6))   # (n, n)
    G, Hs, M = W[2:2 + n, 2:2 + n], W[2:2 + n, 3:3 + n], W[3:3 + n, 2:2 + n]
    b, s = clip1((b1[2:2 + n] + 16) >> 5), clip1((b1[3:3 + n] + 16) >> 5)
    hh, m = clip1((h1[:, 2:2 + n] + 16) >> 5), clip1((h1[:, 3:3 + n] + 16) >> 5)
    j = clip1((j1 + 512) >> 10)

    def avg(p, q):
        return (p + q + 1) >> 1
    return {(0, 0): G, (1, 0): avg(G, b), (2, 0): b, (3, 0): avg(Hs, b),
            (0, 1): avg(G, hh), (1, 1): avg(b, hh), (2, 1): avg(b, j), (3, 1): avg(b, m),
            (0, 2): hh, (1, 2): avg(hh, j), (2, 2): j, (3, 2): avg(j, m),
            (0, 3): avg(M, hh), (1, 3): avg(hh, s), (2, 3): avg(j, s), (3, 3): avg(m, s)}


def chroma_inter(ref, xc0, yc0, mv, n=8, rows=None):
    """8.4.2.2.2 for 4:2:0: the n x n chroma prediction at (xc0, yc0), mv in quarter luma = eighth chroma samples."""
    h, w = ref.shape
    r0, r1 = rows if rows is not None else (0, h - 1)
    xi, yi, fx, fy = xc0 + (mv[0] >> 3), yc0 + (mv[1] >> 3), mv[0] & 7, mv[1] & 7
    ya, yb = np.clip(np.arange(yi, yi + n), r0, r1), np.clip(np.arange(yi + 1, yi + n + 1), r0, r1)
    xa, xb = np.clip(np.arange(xi, xi + n), 0, w - 1), np.clip(np.arange(xi + 1, xi + n + 1), 0, w - 1)
    R = ref.astype(np.int64)
    A, B, C, D = R[np.ix_(ya, xa)], R[np.ix_(ya, xb)], R[np.ix_(yb, xa)], R[np.ix_(yb, xb)]
    return ((8 - fx) * (8 - fy) * A + fx * (8 - fy) * B + (8 - fx) * fy * C + fx * fy * D + 32) >> 6


# ------------------------------------------------------------------------------------------------ motion (§5.3)
def se_bits(v):
    """Length of the se(v) code of v."""
    k = 2 * v - 1 if v > 0 else -2 * v
    return 2 * int(k + 1).bit_length() - 1


def motion_cost(sad, mv, qp):
    """§5.3: SAD + λ(qp)·(bits(mvx) + bits(mvy)), plus 4 bits for a fractional vector (mv in quarter samples)."""
    frac = FRAC_PENALTY_BITS if (mv[0] | mv[1]) & 3 else 0
    return sad + LAMBDA[qp] * (se_bits(mv[0]) + se_bits(mv[1]) + frac)


def sad(a, b):
    return int(np.abs(np.asarray(a, np.int64) - np.asarray(b, np.int64)).sum())


MV_MAX_FULL = 255                # §5.3 vector range, full samples per component (wide-range motion)


def mv_ok(vx, vy):
    """§5.3: a full-sample vector is usable when both components lie in [-255, 255]."""
    return -MV_MAX_FULL <= vx <= MV_MAX_FULL and -MV_MAX_FULL <= vy <= MV_MAX_FULL


def full_search(src_blk, ref, x0, y0, qp, rows=None, centre=(0, 0), dy_range=16):
    """Brute force over the window centred on the full-sample vector `centre` — dx in [-16, 15], dy in [-dy_range, dy_range]
    around it — with clamped coordinates (8.4.2.2.1: a full-sample prediction is the reference sample at the clamped position), the
    vectors outside mv_ok left out: {(vx, vy) full samples: (SAD, cost)}."""
    h, w = ref.shape
    r0, r1 = rows if rows is not None else (0, h - 1)
    cx, cy = centre
    ys = np.clip(np.arange(y0 + cy - 16, y0 + cy + 16 + 16), r0, r1)
    xs = np.clip(np.arange(x0 + cx - 16, x0 + cx + 15 + 16), 0, w - 1)
    win = sliding_window_view(ref[np.ix_(ys, xs)].astype(np.int64), (16, 16))      # win[16 + dy, 16 + dx] = the prediction
    sads = np.abs(win - np.asarray(src_blk, np.int64)).sum(axis=(2, 3))
    out = {}
    for dy in range(-dy_range, dy_range + 1):
        for dx in range(-16, 16):
            v = (cx + dx, cy + dy)
            if mv_ok(*v):
                s = int(sads[16 + dy, 16 + dx])
                out[v] = (s, motion_cost(s, (4 * v[0], 4 * v[1]), qp))
    return out


def search(src_blk, ref, x0, y0, qp, centre=(0, 0), dy_range=16):
    """§5.3: the exhaustive search (dy_range 16), or the reduced one on new content (dy_range 2), in the window centred on `centre`:
    the full-sample vector of the lowest key cost << 11 | (vy − cy + 16)·32 + (vx − cx + 16), so that equal costs go to the lower
    row, then the lower column.  Returns (vector, SAD, cost)."""
    costs = full_search(src_blk, ref, x0, y0, qp, centre=centre, dy_range=dy_range)
    v = min(costs, key=lambda v: (costs[v][1], v[1], v[0]))
    return v, costs[v][0], costs[v][1]


NB8 = [(-1, -1), (0, -1), (1, -1), (-1, 0), (1, 0), (-1, 1), (0, 1), (1, 1)]    # §5.3: the refinement's neighbour order


def refine(src_blk, ref, x0, y0, v, centre, sad_int, qp):
    """§5.3 quarter-sample refinement of the full-sample vector v, found in the window centred on `centre` with SAD sad_int.  The gate:
    |v − centre| ≤ 13 per component (the 6-tap support stays inside the window) and 96·λ < sad_int < 8192; closed, v stands.  Stage H
    scores v and its 8 half-sample neighbours, stage Q the stage-H winner and its 8 quarter-sample neighbours, each by motion_cost
    (SAD + λ·(bits(mvx) + bits(mvy)), 4 bits more when fractional) of the real vector and the lowest (cost, i) wins, i = 0 the
    centre and 1..8 the neighbours in NB8's order: the centre wins ties.  Predictions by 8.4.2.2.1 on the clamped reference.
    Returns (quarter-sample vector, whether the gate was open)."""
    mv = (4 * v[0], 4 * v[1])
    if not (abs(v[0] - centre[0]) <= 13 and abs(v[1] - centre[1]) <= 13
            and EARLY_SAD_PER_LAMBDA * LAMBDA[qp] < sad_int < REFINE_MAX_SAD):
        return mv, False
    planes = luma_planes(ref, x0 + v[0] - 1, y0 + v[1] - 1, 17)       # every offset in [-3, 3] quarter samples around v
    blk = np.asarray(src_blk, np.int64)

    def cost(q):
        ox, oy = q[0] - 4 * v[0] + 4, q[1] - 4 * v[1] + 4             # quarter samples from (v − 1), in [1, 7]
        pred = planes[(ox & 3, oy & 3)][oy >> 2:(oy >> 2) + 16, ox >> 2:(ox >> 2) + 16]
        return motion_cost(sad(blk, pred), q, qp)
    for step in (2, 1):
        cands = [mv] + [(mv[0] + step * i, mv[1] + step * j) for i, j in NB8]
        mv = cands[min(range(9), key=lambda i: (cost(cands[i]), i))]
    return mv, True


def anchor_of(mbx, mby, mbw, band_r0, band_r1):
    """§5.3: the anchor of a macroblock is offset (1, 1) of its 4x4 group, rows counted inside the band [band_r0, band_r1),
    clamped into the band and the picture for partial groups."""
    return min(4 * (mbx // 4) + 1, mbw - 1), min(band_r0 + 4 * ((mby - band_r0) // 4) + 1, band_r1 - 1)


# ------------------------------------------------------------------------------------------------ wide-range motion (§5.3)
COARSE_DX, COARSE_DY = 32, 64    # the coarse search: dx in [-32, 31], dy in [-64, 63] decimated samples


def decimate(y):
    """The decimated luma of a coded luma plane: each sample the rounded mean (s + 8) >> 4 of the sum s of a 4x4 block."""
    y = np.asarray(y, np.int64)
    h, w = y.shape
    return (y.reshape(h // 4, 4, w // 4, 4).sum(axis=(1, 3)) + 8) >> 4


def coarse_search(dec_cur, dec_ref, mbx, mby, mbw, band_r0, band_r1, sad0, qp):
    """The coarse vector (dx, dy) in decimated samples of the anchor group of macroblock (mbx, mby), or None.  Only an anchor whose
    co-located full-resolution SAD `sad0` exceeds 96·λ searches.  The group (4x4 macroblocks, rows counted inside the band
    [band_r0, band_r1), partial at the picture's right edge and the band's bottom) is a decimated block of up to 16x16 samples,
    compared with dec_ref at every dx in [-32, 31], dy in [-64, 63] that keeps it inside the plane and the band's decimated rows;
    the winner is the lexicographic minimum of (SAD, |dx| + |dy|, dy, dx).  The planes are decimate() of whole coded pictures."""
    if anchor_of(mbx, mby, mbw, band_r0, band_r1) != (mbx, mby) or sad0 <= EARLY_SAD_PER_LAMBDA * LAMBDA[qp]:
        return None
    gx0, gy0 = 4 * (mbx // 4), band_r0 + 4 * ((mby - band_r0) // 4)
    X0, Y0, W, H = 4 * gx0, 4 * gy0, 4 * (min(gx0 + 4, mbw) - gx0), 4 * (min(gy0 + 4, band_r1) - gy0)
    blk = np.asarray(dec_cur, np.int64)[Y0:Y0 + H, X0:X0 + W]
    lo, hi, dw = 4 * band_r0, 4 * band_r1, dec_ref.shape[1]
    dxs = [dx for dx in range(-COARSE_DX, COARSE_DX) if 0 <= X0 + dx and X0 + dx + W <= dw]
    dys = [dy for dy in range(-COARSE_DY, COARSE_DY) if lo <= Y0 + dy and Y0 + dy + H <= hi]
    if not dxs or not dys:
        return None
    win = sliding_window_view(np.asarray(dec_ref, np.int64), (H, W))                # win[y, x] = the block at (x, y)
    sads = np.abs(win[Y0 + dys[0]:Y0 + dys[-1] + 1, X0 + dxs[0]:X0 + dxs[-1] + 1] - blk).sum(axis=(2, 3))
    DY, DX = (a.ravel() for a in np.meshgrid(dys, dxs, indexing="ij"))
    i = np.lexsort((DX, DY, np.abs(DX) + np.abs(DY), sads.ravel()))[0]
    return int(DX[i]), int(DY[i])


def second_window(coarse):
    """§5.3: the full-sample centre (coarse × 4) of an anchor's second ±16 search, or None — no coarse vector, or one the co-located
    search covers with the 4 samples either way a decimated sample spans (x in [-12, 11] and y in [-12, 12])."""
    if coarse is None:
        return None
    cx, cy = 4 * coarse[0], 4 * coarse[1]
    return None if -12 <= cx <= 11 and -12 <= cy <= 12 else (cx, cy)


# ------------------------------------------------------------------------------------------------ the lean pass's exits (§5.3, §5.12, §5.13)
PRED_SAD_FACTOR = 4              # §5.3: a temporal predictor is taken with a SAD of at most 4·96·λ
LTR_CHANGED_MIN_DIV, LTR_CHANGED_RATIO = 64, 8      # §5.13: the marking rule


def scale_mv(v, num, den):
    """§5.12: one component of the previous picture's vector, which spanned `den` pictures, as a predictor for a reference `num`
    pictures back: unchanged, doubled, or halved rounding half away from zero."""
    if num == den:
        return v
    if num > den:
        return 2 * v
    return -((-v + 1) >> 1) if v < 0 else (v + 1) >> 1


def full_pred(ref, x0, y0, v):
    """The 16x16 full-sample prediction at (x0, y0) for vector v (full samples), coordinates clamped to the plane (8.4.2.2.1)."""
    h, w = ref.shape
    ys, xs = np.clip(np.arange(y0 + v[1], y0 + v[1] + 16), 0, h - 1), np.clip(np.arange(x0 + v[0], x0 + v[0] + 16), 0, w - 1)
    return ref[np.ix_(ys, xs)].astype(np.int64)


def predictor_candidate(mv, wide):
    """§5.3: the previous vector `mv` (quarter samples, already scaled) rounded to the full-sample candidate k = ((mv + 2) >> 2), and
    the centre of the window its test runs in: (0, 0) when k lies in the co-located window's test range (x in [-15, 14], y in
    [-15, 15], so that its 8 neighbours are in the window too); with wide motion, outside that range and within the vector range,
    the window re-centred on (kx & ~3, ky).  None: the predictor is not tested."""
    k = ((mv[0] + 2) >> 2, (mv[1] + 2) >> 2)
    if -15 <= k[0] <= 14 and -15 <= k[1] <= 15:
        return k, (0, 0)
    if wide and mv_ok(*k):
        return k, (k[0] & ~3, k[1])
    return None


def predictor_test(src_blk, ref, x0, y0, k, centre, sad0, qp):
    """§5.3: the 3x3 test of full-sample candidate k (real vector) in the window centred on `centre`.  Every position's key is
    cost << 11 | index, cost = SAD + λ·(bits(4x) + bits(4y)) of the real vector and index = (y − cy + 16)·32 + (x − cx + 16) relative
    to the window, so equal costs go to the lower row, then the lower column.  Taken when the candidate's SAD ≤ 4·96·λ, its key is
    below all 8 neighbours' (a strict local minimum) and at most the zero vector's key0 = (sad0 + 2λ) << 11 | 528.  Returns the
    candidate's SAD when taken, None otherwise."""
    lam = LAMBDA[qp]
    keys = {}
    for j in (-1, 0, 1):
        for i in (-1, 0, 1):
            v = (k[0] + i, k[1] + j)
            s = sad(src_blk, full_pred(ref, x0, y0, v))
            keys[(i, j)] = (s, (s + lam * (se_bits(4 * v[0]) + se_bits(4 * v[1]))) << 11 | (v[1] - centre[1] + 16) * 32 + (v[0] - centre[0] + 16))
    sadc, kc = keys.pop((0, 0))
    key0 = (sad0 + 2 * lam) << 11 | (16 * 32 + 16)
    taken = sadc <= PRED_SAD_FACTOR * EARLY_SAD_PER_LAMBDA * lam and all(kc < kk for _, kk in keys.values()) and kc <= key0
    return sadc if taken else None


class Exit:
    """The lean pass's class of one macroblock (lean_exit).  cls: "zero", "predictor", "long-term" or "searched".  k: the
    predictor's full-sample candidate (or None); frac: the previous vector was fractional; lean: the lean pass took the predictor
    (otherwise the search pass did, on the clamped window, with its refinement).  For decide(): sad0, the co-located SAD; tried,
    the temporal predictor's candidate when it was tested (hit or not); centre and sad, the window and the SAD of a hit."""

    def __init__(self, cls, k=None, frac=False, lean=False, search_pred=False, sad0=0, tried=None, centre=(0, 0), sad=0):
        self.cls, self.k, self.frac, self.lean = cls, k, frac, lean
        self.search_pred = search_pred          # "long-term": the search pass's predictor test would have hit
        self.sad0, self.tried, self.centre, self.sad = sad0, tried, centre, sad


def lean_exit(src_blk, ref, lt, prev, x0, y0, qp, wide=False, dist=(1, 1)):
    """§5.3 / §5.12 / §5.13: the class of the macroblock at (x0, y0) with source luma `src_blk`.  ref: the model's reconstruction of
    refIdx 0 (luma); lt: the long-term picture's (None while there is none); prev: the previous picture's parsed record at this
    address (None after nothing); dist: (ref_dist, prev_ref_dist) of §5.12.
      1. zero: SAD(0,0) ≤ 96·λ.
      2. the temporal predictor: only a P macroblock record (P_Skip included; intra and I_PCM give none) gives one, its vector scaled
         by dist and rounded (predictor_candidate), tested by predictor_test.  The lean pass takes a hit only when the window's 48
         columns lie inside the picture (x0 − 16 + cx ≥ 0, x0 + 32 + cx ≤ width) and the previous vector was full-sample; a hit of
         a picture-edge macroblock or of a fractional previous vector is the search pass's, on the clamped window (the same test).
      3. long-term: while there is a long-term picture, its SAD at the zero vector ≤ 96·λ — tried in the lean pass only, so only
         when 1 and the lean pass's part of 2 failed: an edge or fractional-vector macroblock whose search-pass predictor would hit
         takes the long-term picture, an inside one whose lean predictor hits never tries it.
      4. searched: the search passes, with the search pass's predictor hit when there is one."""
    lam = LAMBDA[qp]
    thr = EARLY_SAD_PER_LAMBDA * lam
    sad0 = sad(src_blk, full_pred(ref, x0, y0, (0, 0)))
    if sad0 <= thr:
        return Exit("zero", sad0=sad0)
    hit, tried = None, None
    if prev is not None and prev.kind in ("P_L0_16x16", "P_Skip"):
        mv = tuple(scale_mv(c, *dist) for c in prev.mv)
        cand = predictor_candidate(mv, wide)
        if cand is not None:
            tried = cand[0]
            s = predictor_test(src_blk, ref, x0, y0, cand[0], cand[1], sad0, qp)
            if s is not None:
                inside = x0 - 16 + cand[1][0] >= 0 and x0 + 32 + cand[1][0] <= ref.shape[1]
                hit = cand, bool((mv[0] | mv[1]) & 3), inside, s
    if hit is not None and hit[2] and not hit[1]:
        return Exit("predictor", hit[0][0], False, lean=True, sad0=sad0, tried=tried, centre=hit[0][1], sad=hit[3])
    if lt is not None and sad(src_blk, full_pred(lt, x0, y0, (0, 0))) <= thr:
        return Exit("long-term", search_pred=hit is not None, sad0=sad0, tried=tried)
    if hit is not None:
        return Exit("predictor", hit[0][0], hit[1], lean=False, sad0=sad0, tried=tried, centre=hit[0][1], sad=hit[3])
    return Exit("searched", sad0=sad0, tried=tried)


class Decision:
    """What §5.3 decides for one macroblock: ref_idx and mv (quarter samples) — what it is coded with unless the I_PCM rule of §5.7
    sends it raw; ex, its lean_exit; path, how the vector was found: "zero", "long-term", "predictor" (the temporal predictor),
    "anchor predictor", "search" or "reduced search"; full, centre and sad: the full-sample vector before refinement, the centre of
    its window and its SAD; src: the vector a predictor hit came from; refined, the refinement's gate was open; second, the anchor's
    second window won; bad, the new-content flag an anchor publishes with its vector."""

    def __init__(self, ex, path, ref_idx=0, mv=(0, 0), full=(0, 0), centre=(0, 0), sad=0, src=None, refined=False, second=False):
        self.ex, self.path, self.ref_idx, self.mv = ex, path, ref_idx, mv
        self.full, self.centre, self.sad, self.src = full, centre, sad, src
        self.refined, self.second = refined, second
        self.bad = path not in ("zero", "long-term") and sad >= REFINE_MAX_SAD


def decide(src_blk, ref, lt, prev, x0, y0, qp, wide=False, dist=(1, 1), anchor=None, coarse=None):
    """§5.3 / §5.12 / §5.13: the final refIdx and vector of the macroblock at (x0, y0), after lean_exit (same arguments).  anchor:
    the Decision of the macroblock's anchor (None: the macroblock is an anchor; anchors are decided first); coarse: for a wide-motion
    anchor, its group's coarse vector (coarse_search).
      - zero: (0, 0).  long-term: refIdx 1, (0, 0); an anchor publishes the zero vector with the new-content flag clear.
      - a temporal-predictor hit: its candidate k, refined (refine) when the previous vector was fractional.
      - otherwise, a macroblock that is no anchor tests its anchor's vector v the same way (predictor_candidate(v), predictor_test),
        except that the zero vector is not tested twice: a zero candidate is skipped when the temporal predictor tested zero.  A hit
        is refined when v is fractional.  A miss, with the anchor's new-content flag set and SAD(0,0) ≥ 8192, shrinks the search to
        dy in [-2, 2] (the reduced search).
      - otherwise the search of the co-located window, refined; for a wide-motion anchor, also the search of the window centred on
        second_window(coarse) when there is one, which wins when its cost is lower (equal: the co-located window), refined in its
        window.
    The new-content flag: the full-sample SAD of the vector before refinement ≥ 8192 for a hit or a search, clear for the zero and
    long-term exits."""
    ex = lean_exit(src_blk, ref, lt, prev, x0, y0, qp, wide, dist)
    if ex.cls == "zero":
        return Decision(ex, "zero")
    if ex.cls == "long-term":
        return Decision(ex, "long-term", ref_idx=1)

    def hit(path, k, centre, s, src):
        frac = bool((src[0] | src[1]) & 3)
        mv, refined = refine(src_blk, ref, x0, y0, k, centre, s, qp) if frac else ((4 * k[0], 4 * k[1]), False)
        return Decision(ex, path, mv=mv, full=k, centre=centre, sad=s, src=src, refined=refined)
    if ex.cls == "predictor":
        return hit("predictor", ex.k, ex.centre, ex.sad, tuple(scale_mv(c, *dist) for c in prev.mv))
    dy_range = 16
    if anchor is not None:
        cand = predictor_candidate(anchor.mv, wide)
        if cand is not None and not (cand[0] == (0, 0) and ex.tried == (0, 0)):
            s = predictor_test(src_blk, ref, x0, y0, cand[0], cand[1], ex.sad0, qp)
            if s is not None:
                return hit("anchor predictor", cand[0], cand[1], s, anchor.mv)
        if anchor.bad and ex.sad0 >= REFINE_MAX_SAD:
            dy_range = 2
    v, s, c = search(src_blk, ref, x0, y0, qp, dy_range=dy_range)
    centre, second = (0, 0), False
    far = second_window(coarse) if wide and anchor is None else None
    if far is not None:
        v2, s2, c2 = search(src_blk, ref, x0, y0, qp, centre=far)
        if c2 < c:
            v, s, centre, second = v2, s2, far, True
    mv, refined = refine(src_blk, ref, x0, y0, v, centre, s, qp)
    return Decision(ex, "search" if dy_range == 16 else "reduced search", mv=mv, full=v, centre=centre, sad=s, refined=refined,
                    second=second)


def changed_count(src_y, ref_y, qp):
    """§5.13 changed(k): the macroblocks of a P picture whose co-located SAD against its short-term reference fails the zero-motion
    exit (> 96·λ), counted from the source luma and the model's reconstruction of the reference."""
    h, w = src_y.shape
    d = np.abs(np.asarray(src_y, np.int64) - np.asarray(ref_y, np.int64)).reshape(h // 16, 16, w // 16, 16).sum(axis=(1, 3))
    return int((d > EARLY_SAD_PER_LAMBDA * LAMBDA[qp]).sum())


def marks(changed, changed_prev, mbs):
    """§5.13: picture k marks picture k − 1 long-term when changed(k) ≥ max(⌈mbs/64⌉, 8·changed(k−1)) (an IDR counts every macroblock)."""
    return changed >= max(-(-mbs // LTR_CHANGED_MIN_DIV), LTR_CHANGED_RATIO * changed_prev)


def marking_ops(long_term_exists):
    """§5.13: the operations of a marking picture — MMCO 1 on the picture two back only while there is no long-term picture (the
    sliding window holds two short-term frames then), MMCO 4 (one long-term index), MMCO 3 (the previous picture to index 0)."""
    return ([] if long_term_exists else [(1, 1)]) + [(4, 1), (3, 0, 0)]


# ------------------------------------------------------------------------------------------------ the intra decision (§5.2, §5.7)
I4_SKIP_SAD_PER_LAMBDA = 32      # §5.2: Intra4x4 is tried only when the best Intra16x16 SAD exceeds 32·λ
MB_BITS_LIMIT = 3200             # A.3.1 / §5.7: a macroblock sized above this is sent as I_PCM


def rd_lambda(qp):
    """§5.2: the Lagrangian of the Intra4x4 / Intra16x16 choice, round(0.85·2^((qp − 12)/3)), at least 1."""
    return max(1, int(np.floor(0.85 * 2.0 ** ((qp - 12) / 3) + 0.5)))


def _blocks(x):
    """(..., 16, 16) -> (..., 16 blkIdx, 4, 4): the 4x4 luma blocks of a macroblock in decoding order."""
    x = np.asarray(x, np.int64)
    b = x.reshape(*x.shape[:-2], 4, 4, 4, 4).swapaxes(-3, -2)           # [..., by, bx, r, c]
    return np.stack([b[..., by, bx, :, :] for bx, by in BLK_XY], axis=-3)


def _unblocks(b):
    """_blocks' inverse."""
    out = np.zeros((*b.shape[:-3], 4, 4, 4, 4), np.int64)
    for blk, (bx, by) in enumerate(BLK_XY):
        out[..., by, bx, :, :] = b[..., blk, :, :]
    return out.swapaxes(-3, -2).reshape(*b.shape[:-3], 16, 16)


def _chroma_blocks(x):
    """(..., 8, 8) -> (..., 4, 4, 4): the 4x4 blocks of one chroma component, raster order (= chroma4x4BlkIdx)."""
    x = np.asarray(x, np.int64)
    return x.reshape(*x.shape[:-2], 2, 4, 2, 4).swapaxes(-3, -2).reshape(*x.shape[:-2], 4, 4, 4)


def _chroma_unblocks(b):
    return b.reshape(*b.shape[:-3], 2, 2, 4, 4).swapaxes(-3, -2).reshape(*b.shape[:-3], 8, 8)


def chroma_code(src, pred, qpc, intra):
    """§5.4 for one chroma component of a stack of macroblocks ((N, 8, 8) source and prediction): (DC levels (N, 4), AC levels
    (N, 4, 16) in scan order, position 0 unused, the reconstruction (N, 8, 8))."""
    pb = _chroma_blocks(pred)
    lv, w = quant_block(_chroma_blocks(src) - pb, qpc, intra, with_dc=False)
    n = lv.shape[0]
    dc = chroma_dc_levels(w[..., 0, 0].reshape(n, 2, 2), qpc, intra)
    d = dequant4x4(lv, qpc)
    d[..., 0, 0] = chroma_dc_dequant(dc, qpc).reshape(n, 4)
    return dc.reshape(n, 4), raster_to_scan(lv), _chroma_unblocks(clip1(pb + inverse4x4(d)))


def chroma_bits(dcs, acs):
    """§5.7: the chroma bits of one macroblock from its two components' DC (4) and AC (4, 16) levels, and its coded_block_pattern
    chroma part: 2 when an AC level is non-zero, 1 when only a DC level is."""
    cc = 2 if any(np.any(a[:, 1:]) for a in acs) else 1 if any(np.any(d) for d in dcs) else 0
    bits = sum(cavlc_bits(d, chroma_dc=True) for d in dcs) if cc else 0
    if cc == 2:
        bits += sum(cavlc_bits(a[b][1:]) for a in acs for b in range(4))
    return bits, cc


class IntraDecision:
    """intra_decide's result for a stack of N macroblocks (arrays of N): kind ("I_16x16", "I_NxN" or "I_PCM"); i16_mode and
    chroma_mode; i4_modes (N, 16) by blkIdx, those of the Intra4x4 pass; tried, the gate let Intra4x4 be tried; j16, j4 (the model
    runs the Intra4x4 pass everywhere, so that j4 < j16 where it was not tried shows what the gate decided); size, the §5.7 size of the kind the comparison kept; i16_tie / chroma_tie, the two modes' SADs were
    equal; rec, the reconstruction (Y (N, 16, 16), Cb, Cr (N, 8, 8)); right, what the next macroblock takes as its left neighbour."""


def intra_decide(src_y, src_u, src_v, left, qp):
    """§5.2: the intra decision of N macroblocks that have no neighbour above (src_y (N, 16, 16), src_u / src_v (N, 8, 8)).  left:
    None at a slice start, else (y (N, 16), cb (N, 8), cr (N, 8), modes (N, 4)): the left neighbour's reconstructed right column and
    the Intra4x4PredMode of its right-column blocks (2 where it is not I_NxN).
      - Intra16x16: argmin of SAD·4 + mode over horizontal (1, with a left neighbour) and DC (2).
      - chroma: argmin of (SAD Cb + SAD Cr)·4 + mode over DC (0) and horizontal (1, with a left neighbour).
      - Intra4x4 is tried when the best Intra16x16 SAD exceeds 32·λ: per block in decoding order the key
        (SAD + λ·(mode == predIntra4x4PredMode ? 1 : 4))·16 + mode over the modes whose samples are available, the block reconstructed
        before the next is predicted.
      - J = SSD(source, reconstruction) + rd_lambda(qp)·bits over the luma: Intra16x16 8 + the DC block + the 15-coefficient blocks
        when any AC level is non-zero, Intra4x4 8 + the blocks of its cbp + its mode bits (1 or 4 per block), blocks by cavlc_bits;
        Intra4x4 wins when its J is strictly smaller.
      - §5.7: I_PCM when header_budget (48, 96 for I_NxN) + luma bits + chroma bits > 3200."""
    sy, su, sv = (np.asarray(a, np.int64) for a in (src_y, src_u, src_v))
    n, idx = sy.shape[0], np.arange(sy.shape[0])
    lam, rdl, qpc = LAMBDA[qp], rd_lambda(qp), QPC[qp]
    has_left = left is not None
    ly, lu, lv_, lmodes = (np.asarray(a, np.int64) for a in left) if has_left else (None,) * 4
    out = IntraDecision()
    # ---- Intra16x16 mode
    m16 = ([1] if has_left else []) + [2]
    p16 = np.stack([np.stack([intra16_pred(m, None, None if ly is None else ly[i], None) for i in range(n)]) for m in m16])
    sad16 = np.abs(sy - p16).sum(axis=(2, 3))
    k = (sad16 * 4 + np.array(m16)[:, None]).argmin(0)
    out.i16_mode, pred16 = np.array(m16)[k], p16[k, idx]
    best16 = sad16[k, idx]
    out.i16_tie = sad16[0] == sad16[1] if has_left else np.zeros(n, bool)
    # ---- chroma mode
    mc = [0] + ([1] if has_left else [])
    pc = np.stack([np.stack([np.stack([chroma_pred(m, None, None if l_ is None else l_[i], None) for i in range(n)])
                             for l_ in ((lu, lv_) if has_left else (None, None))]) for m in mc])       # (modes, 2, N, 8, 8)
    sadc = (np.abs(np.stack([su, sv]) - pc).sum(axis=(3, 4))).sum(axis=1)
    kc = (sadc * 4 + np.array(mc)[:, None]).argmin(0)
    out.chroma_mode = np.array(mc)[kc]
    out.chroma_tie = sadc[0] == sadc[1] if has_left else np.zeros(n, bool)
    cbits = np.zeros(n, np.int64)
    coded_c = [chroma_code(s_, pc[kc, c, idx], qpc, True) for c, s_ in enumerate((su, sv))]
    for i in range(n):
        cbits[i] = chroma_bits([coded_c[0][0][i], coded_c[1][0][i]], [coded_c[0][1][i], coded_c[1][1][i]])[0]
    crec = [coded_c[0][2], coded_c[1][2]]
    # ---- Intra16x16 coding
    pb = _blocks(pred16)
    lv, w = quant_block(_blocks(sy) - pb, qp, True, with_dc=False)
    w_dc = np.zeros((n, 4, 4), np.int64)
    for blk, (bx, by) in enumerate(BLK_XY):
        w_dc[:, by, bx] = w[:, blk, 0, 0]
    dc = i16_dc_levels(w_dc, qp)
    dcy = luma_dc_dequant(dc, qp)
    d = dequant4x4(lv, qp)
    for blk, (bx, by) in enumerate(BLK_XY):
        d[:, blk, 0, 0] = dcy[:, by, bx]
    rec16 = _unblocks(clip1(pb + inverse4x4(d)))
    ac, dcs = raster_to_scan(lv), raster_to_scan(dc)
    bits16 = np.array([cavlc_bits(dcs[i]) + (sum(cavlc_bits(ac[i, b, 1:]) for b in range(16)) if np.any(ac[i]) else 0)
                       for i in range(n)])
    out.j16 = ((sy - rec16) ** 2).sum(axis=(1, 2)) + rdl * (8 + bits16)
    # ---- Intra4x4: the gate, and the pass (on every macroblock)
    out.tried = best16 > I4_SKIP_SAD_PER_LAMBDA * lam
    rt = np.zeros((n, 17, 17), np.int64)            # rt[:, 1 + y, 1 + x]: sample (x, y) of the macroblock; column 0 the left one
    if has_left:
        rt[:, 1:, 0] = ly
    av = Avail(has_left, False, False, False)
    levels, modes, mode_bits = np.zeros((n, 16, 16), np.int64), np.zeros((n, 16), np.int64), np.zeros(n, np.int64)
    for blk, (bx, by) in enumerate(BLK_XY):
        P = intra4x4_accessor(lambda nx, ny: rt[:, 1 + ny, 1 + nx], blk, av)
        cands, preds = [], []
        for mode in range(9):
            try:
                preds.append(np.broadcast_to(intra4x4_pred(mode, P), (n, 4, 4)))
                cands.append(mode)
            except (ValueError, TypeError):          # the mode reads a sample that is not available
                pass
        if by == 0 or (bx == 0 and not has_left):    # 8.3.1.1: block A or B not available
            pm = np.full(n, 2)
        else:
            ma = modes[:, BLK_IDX[(bx - 1, by)]] if bx > 0 else lmodes[:, by]
            pm = np.minimum(ma, modes[:, BLK_IDX[(bx, by - 1)]])
        src = sy[:, 4 * by:4 * by + 4, 4 * bx:4 * bx + 4]
        keys = np.stack([(np.abs(src - p).sum(axis=(1, 2)) + lam * np.where(pm == m, 1, 4)) * 16 + m for m, p in zip(cands, preds)])
        kk = keys.argmin(0)
        mode, pred = np.array(cands)[kk], np.stack(preds)[kk, idx]
        l4, _ = quant_block(src - pred, qp, True)
        levels[:, blk], modes[:, blk] = raster_to_scan(l4), mode
        mode_bits += np.where(mode == pm, 1, 4)
        rt[:, 1 + 4 * by:5 + 4 * by, 1 + 4 * bx:5 + 4 * bx] = clip1(pred + inverse4x4(dequant4x4(l4, qp)))
    bits4 = np.array([sum(cavlc_bits(levels[i, b]) for b in range(16) if np.any(levels[i, b & ~3:(b & ~3) + 4])) for i in range(n)])
    rec4 = rt[:, 1:, 1:]
    out.i4_modes = modes
    out.j4 = ((sy - rec4) ** 2).sum(axis=(1, 2)) + rdl * (8 + bits4 + mode_bits)
    use4 = out.tried & (out.j4 < out.j16)
    out.size = np.where(use4, 2 * HEADER_BITS + bits4, HEADER_BITS + bits16) + cbits
    pcm = out.size > MB_BITS_LIMIT
    out.kind = np.where(pcm, "I_PCM", np.where(use4, "I_NxN", "I_16x16"))
    ry = np.where(pcm[:, None, None], sy, np.where(use4[:, None, None], rec4, rec16))
    ru, rv = (np.where(pcm[:, None, None], s_, r_) for s_, r_ in zip((su, sv), crec))
    out.rec = (ry, ru, rv)
    right_modes = np.full((n, 4), 2, np.int64)
    nxn = out.kind == "I_NxN"
    right_modes[nxn] = out.i4_modes[nxn][:, [BLK_IDX[(3, by)] for by in range(4)]]
    out.right = (ry[:, :, 15], ru[:, :, 7], rv[:, :, 7], right_modes)
    return out


def intra_picture(src, slice_of, mbw, mbh, qp):
    """§5.2 over a whole intra picture whose slices (slice_of[addr]: the slice of each macroblock) never span rows: the macroblocks
    of all slices at the same position in their slice are decided together, each from the model's own reconstruction of its left
    neighbour.  src: (Y, Cb, Cr) planes.  Returns ({addr: (IntraDecision, its index in the stack)}, at_slice_start {addr}, the
    reconstruction (Y, Cb, Cr))."""
    sy, su, sv = (np.asarray(p, np.int64) for p in src)
    chains = {}
    for a in range(mbw * mbh):
        if a % mbw and slice_of[a - 1] == slice_of[a]:
            chains[a] = chains.pop(a - 1) + [a]
        else:
            chains[a] = [a]
    chains = list(chains.values())
    rec = [np.zeros_like(sy), np.zeros_like(su), np.zeros_like(sv)]
    out, left = {}, None
    for j in range(max(len(c) for c in chains)):
        live = [c for c in chains if len(c) > j]
        addrs = [c[j] for c in live]
        ys = np.stack([sy[16 * (a // mbw):16 * (a // mbw) + 16, 16 * (a % mbw):16 * (a % mbw) + 16] for a in addrs])
        us, vs = (np.stack([p[8 * (a // mbw):8 * (a // mbw) + 8, 8 * (a % mbw):8 * (a % mbw) + 8] for a in addrs]) for p in (su, sv))
        if j:
            keep = [i for i, c in enumerate(prev_live) if len(c) > j]
            left = tuple(x[keep] for x in left)
        r = intra_decide(ys, us, vs, left, qp)
        for i, a in enumerate(addrs):
            out[a] = (r, i)
            y0, x0 = 16 * (a // mbw), 16 * (a % mbw)
            rec[0][y0:y0 + 16, x0:x0 + 16] = r.rec[0][i]
            for c in (1, 2):
                rec[c][y0 // 2:y0 // 2 + 8, x0 // 2:x0 // 2 + 8] = r.rec[c][i]
        left, prev_live = r.right, live
    return out, rec


def p_mb_size(src, ref, x0, y0, mv, qp, wide=False):
    """§5.7 / §5.4: the size of the P macroblock at (x0, y0) predicted from the reference planes `ref` (Y, Cb, Cr) at the quarter-
    sample vector mv: its luma levels (dead zone of inter blocks, decimated) and chroma levels quantised by the model, the blocks its
    cbp codes by cavlc_bits, plus 48 (and WM_MVD_BITS with wide motion).  Above 3200 the macroblock is I_PCM."""
    sy, su, sv = (np.asarray(p, np.int64) for p in src)
    pred = luma_inter(ref[0], x0, y0, mv)
    lv, _ = quant_block(_blocks(sy - pred), qp, False)
    scan = decimate_levels(raster_to_scan(lv))
    bits = HEADER_BITS + (WM_MVD_BITS if wide else 0)
    bits += sum(cavlc_bits(scan[b]) for b in range(16) if np.any(scan[b & ~3:(b & ~3) + 4]))
    qpc, coded = QPC[qp], []
    for c, s_ in ((1, su), (2, sv)):
        pc = chroma_inter(ref[c], x0 // 2, y0 // 2, mv)
        dc, ac, _ = chroma_code(s_[None], pc[None], qpc, False)
        coded.append((dc[0], ac[0]))
    return bits + chroma_bits([d for d, _ in coded], [a for _, a in coded])[0]
