"""An independent reader of the Constrained-Baseline CAVLC subset the encoders emit (ITU-T H.264 clauses 7.3, 7.4, 8.3.1.1,
8.4.1, 9.1, 9.2), written from the Recommendation.  It shares no code with oracle/ or selkies_b200/; only the CAVLC code tables
are loaded from oracle/h264_tables_ref.h, which tests/test_h264_tables.py pins byte for byte against libavcodec.

`parse_stream(aus)` returns, per access unit, the SPS in force and one `Mb` record per macroblock in raster order, with the
levels of every block, the derived Intra4x4 modes and motion vector, and the bit length of its macroblock_layer()."""
from __future__ import annotations

import os
from dataclasses import dataclass, field

import numpy as np

from tests.test_h264_tables import parse_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# 8.5.6 frame zig-zag scan: scan index -> (x, y) inside the 4x4 block
ZIGZAG_XY = [(0, 0), (1, 0), (0, 1), (0, 2), (1, 1), (2, 0), (3, 0), (2, 1),
             (1, 2), (0, 3), (1, 3), (2, 2), (3, 1), (3, 2), (2, 3), (3, 3)]
# 6.4.3: luma4x4BlkIdx -> (x, y) of the block in 4-sample units
BLK_XY = [((i >> 2 & 1) * 2 + (i & 1), (i >> 3) * 2 + (i >> 1 & 1)) for i in range(16)]
BLK_IDX = {xy: i for i, xy in enumerate(BLK_XY)}


def _vlc_tables():
    t = parse_tables(os.path.join(ROOT, "oracle", "h264_tables_ref.h"))

    def code(n, v):
        return format(v, f"0{n}b")
    coeff = []
    for tab in range(4):
        d = {}
        for i in range(68):
            n = t["coeff_token_len"][tab][i]
            if n:
                d[code(n, t["coeff_token_bits"][tab][i])] = (i >> 2, i & 3)
        coeff.append(d)
    cdc = {code(n, b): (i >> 2, i & 3) for i, (n, b) in enumerate(zip(t["chroma_dc_coeff_token_len"], t["chroma_dc_coeff_token_bits"])) if n}
    tz = [{code(n, b): z for z, (n, b) in enumerate(zip(ln, bt)) if n} for ln, bt in zip(t["total_zeros_len"], t["total_zeros_bits"])]
    tzc = [{code(n, b): z for z, (n, b) in enumerate(zip(ln, bt)) if n} for ln, bt in zip(t["chroma_dc_total_zeros_len"], t["chroma_dc_total_zeros_bits"])]
    run = [{code(n, b): r for r, (n, b) in enumerate(zip(ln, bt)) if n} for ln, bt in zip(t["run_len"], t["run_bits"])]
    cbp_intra, cbp_inter = [0] * 48, [0] * 48
    for cbp, k in enumerate(t["cbp_to_codenum_intra"]):
        cbp_intra[k] = cbp
    for cbp, k in enumerate(t["cbp_to_codenum_inter"]):
        cbp_inter[k] = cbp
    return coeff, cdc, tz, tzc, run, cbp_intra, cbp_inter


COEFF_TOKEN, CDC_TOKEN, TOTAL_ZEROS, CDC_TOTAL_ZEROS, RUN_BEFORE, CBP_INTRA, CBP_INTER = _vlc_tables()


class SyntaxError_(ValueError):
    pass


# ------------------------------------------------------------------------------------------------ Annex B, 7.3.1, 7.4.1
def split_annexb(au: bytes):
    """NAL units of one Annex-B access unit (start codes 00 00 01 / 00 00 00 01), without their start codes."""
    out, i = [], au.find(b"\x00\x00\x01")
    while i >= 0:
        j = au.find(b"\x00\x00\x01", i + 3)
        nal = au[i + 3: j if j >= 0 else len(au)]
        out.append(nal.rstrip(b"\x00") if j >= 0 else nal)
        i = j
    return out


def unescape(nal: bytes) -> bytes:
    """RBSP of a NAL unit (header byte removed): every 00 00 03 loses its emulation_prevention_three_byte."""
    out, zeros = bytearray(), 0
    for b in nal[1:]:
        if zeros >= 2 and b == 3:
            zeros = 0
            continue
        out.append(b)
        zeros = zeros + 1 if b == 0 else 0
    return bytes(out)


class Bits:
    """MSB-first reader over an RBSP held as a string of '0' / '1'."""

    def __init__(self, rbsp: bytes):
        self.s = "".join(format(b, "08b") for b in rbsp)
        self.pos = 0
        self.end = self.s.rfind("1")             # rbsp_stop_one_bit

    def u(self, n):
        if n == 0:
            return 0
        if self.pos + n > len(self.s):
            raise SyntaxError_("read past the end of the RBSP")
        v = int(self.s[self.pos: self.pos + n], 2)
        self.pos += n
        return v

    def ue(self):                                # 9.1
        z = self.s.find("1", self.pos)
        if z < 0 or z - self.pos > 31:
            raise SyntaxError_("bad Exp-Golomb code")
        n = z - self.pos
        self.pos = z + 1
        return (1 << n) - 1 + self.u(n)

    def se(self):                                # 9.1.1
        k = self.ue()
        return (k + 1) // 2 if k & 1 else -(k // 2)

    def vlc(self, table, maxlen=16):
        for n in range(1, maxlen + 1):
            v = table.get(self.s[self.pos: self.pos + n])
            if v is not None:
                self.pos += n
                return v
        raise SyntaxError_("no VLC code matches")

    def more_rbsp_data(self):
        return self.pos < self.end

    def byte_aligned(self):
        return self.pos % 8 == 0


# ------------------------------------------------------------------------------------------------ 7.3.2.1 SPS, 7.3.2.2 PPS
@dataclass
class Sps:
    profile_idc: int
    constraint_flags: int
    level_idc: int
    log2_max_frame_num: int
    poc_type: int
    max_num_ref_frames: int
    mbw: int
    mbh: int
    crop: tuple          # left, right, top, bottom in chroma-sample units (x2 for luma)
    vui: dict

    @property
    def width(self):
        return self.mbw * 16 - 2 * (self.crop[0] + self.crop[1])

    @property
    def height(self):
        return self.mbh * 16 - 2 * (self.crop[2] + self.crop[3])


def parse_sps(rbsp: bytes) -> Sps:
    b = Bits(rbsp)
    profile, flags, level = b.u(8), b.u(8), b.u(8)
    b.ue()                                               # seq_parameter_set_id
    if profile in (100, 110, 122, 244, 44, 83, 86, 118, 128, 138, 139, 134, 135):
        raise SyntaxError_(f"profile_idc {profile} is outside the subset")
    log2_fn = b.ue() + 4
    poc_type = b.ue()
    if poc_type == 0:
        b.ue()
    elif poc_type == 1:
        raise SyntaxError_("pic_order_cnt_type 1 is outside the subset")
    refs = b.ue()
    b.u(1)                                               # gaps_in_frame_num_value_allowed_flag
    mbw, mbh = b.ue() + 1, b.ue() + 1
    if not b.u(1):
        raise SyntaxError_("field coding is outside the subset")
    b.u(1)                                               # direct_8x8_inference_flag
    crop = (b.ue(), b.ue(), b.ue(), b.ue()) if b.u(1) else (0, 0, 0, 0)
    vui = {}
    if b.u(1):                                           # E.1.1
        if b.u(1):
            idc = b.u(8)
            vui["aspect_ratio_idc"] = idc
            if idc == 255:
                b.u(32)
        if b.u(1):
            vui["overscan_appropriate"] = b.u(1)
        if b.u(1):
            vui["video_format"], vui["video_full_range_flag"] = b.u(3), b.u(1)
            if b.u(1):
                vui["colour_primaries"], vui["transfer_characteristics"], vui["matrix_coefficients"] = b.u(8), b.u(8), b.u(8)
        if b.u(1):
            vui["chroma_sample_loc_type_top"], vui["chroma_sample_loc_type_bottom"] = b.ue(), b.ue()
        vui["timing_info_present_flag"] = b.u(1)
        if vui["timing_info_present_flag"]:
            b.u(32), b.u(32), b.u(1)
        vui["nal_hrd"], vui["vcl_hrd"] = b.u(1), 0
        if vui["nal_hrd"]:
            raise SyntaxError_("HRD parameters are outside the subset")
        vui["vcl_hrd"] = b.u(1)
        if vui["vcl_hrd"]:
            raise SyntaxError_("HRD parameters are outside the subset")
        vui["pic_struct_present_flag"] = b.u(1)
        if b.u(1):
            vui["motion_vectors_over_pic_boundaries_flag"] = b.u(1)
            vui["max_bytes_per_pic_denom"], vui["max_bits_per_mb_denom"] = b.ue(), b.ue()
            vui["log2_max_mv_length_horizontal"], vui["log2_max_mv_length_vertical"] = b.ue(), b.ue()
            vui["max_num_reorder_frames"], vui["max_dec_frame_buffering"] = b.ue(), b.ue()
    if b.pos != b.end:
        raise SyntaxError_("SPS does not end in rbsp_trailing_bits")
    return Sps(profile, flags, level, log2_fn, poc_type, refs, mbw, mbh, crop, vui)


def parse_pps(rbsp: bytes) -> dict:
    b = Bits(rbsp)
    p = dict(pps_id=b.ue(), sps_id=b.ue(), entropy_coding_mode_flag=b.u(1), bottom_field_pic_order=b.u(1),
             num_slice_groups=b.ue() + 1, num_ref_idx_l0=b.ue() + 1, num_ref_idx_l1=b.ue() + 1, weighted_pred_flag=b.u(1),
             weighted_bipred_idc=b.u(2), pic_init_qp=26 + b.se(), pic_init_qs=26 + b.se(), chroma_qp_index_offset=b.se(),
             deblocking_filter_control_present_flag=b.u(1), constrained_intra_pred_flag=b.u(1), redundant_pic_cnt_present_flag=b.u(1))
    if p["entropy_coding_mode_flag"] or p["num_slice_groups"] != 1 or p["weighted_pred_flag"] or p["redundant_pic_cnt_present_flag"]:
        raise SyntaxError_("PPS outside the Constrained-Baseline CAVLC subset")
    if b.pos != b.end:
        raise SyntaxError_("PPS carries High-profile extensions")
    return p


# ------------------------------------------------------------------------------------------------ macroblock records
@dataclass
class Mb:
    addr: int
    slice: int                   # index of the slice inside the picture
    kind: str                    # "I_NxN", "I_16x16", "I_PCM", "P_L0_16x16", "P_Skip"
    qp: int
    cbp: int = 0                 # luma bits 0..3 (8x8 quadrants), chroma << 4
    i16_mode: int = -1
    chroma_mode: int = -1
    i4_modes: list = None        # Intra4x4PredMode per luma4x4BlkIdx
    mv: tuple = (0, 0)           # quarter-sample units
    mvd: tuple = (0, 0)
    luma_dc: np.ndarray = None   # Intra16x16DCLevel, scan order (16)
    luma: np.ndarray = None      # (16 blkIdx, 16 scan positions); position 0 unused for Intra16x16
    chroma_dc: np.ndarray = None  # (2, 4)
    chroma_ac: np.ndarray = None  # (2, 4 blkIdx, 16 scan positions); position 0 unused
    total_coeff: np.ndarray = None   # luma TotalCoeff per blkIdx (16 for I_PCM, 0 for P_Skip)
    total_coeff_c: np.ndarray = None  # (2, 4)
    pcm: tuple = None            # (luma 16x16, cb 8x8, cr 8x8) uint8
    bits: int = 0                # length of macroblock_layer() (0 for P_Skip)
    skip_mv: tuple = None        # P_L0_16x16: the vector a P_Skip would have inferred here (8.4.1.1)

    @property
    def intra(self):
        return self.kind.startswith("I")

    def luma_raster(self, blk):
        """Levels of luma block `blk` as a 4x4 raster array."""
        return scan_to_raster(self.luma[blk])


def scan_to_raster(levels):
    out = np.zeros((4, 4), np.int64)
    for k, (x, y) in enumerate(ZIGZAG_XY):
        out[y, x] = levels[k]
    return out


@dataclass
class Picture:
    sps: Sps
    idr: bool
    frame_num: int
    qp: int                      # slice QP of the first slice
    nal_ref_idc: int = 1         # of the first slice: 0 for a non-reference picture
    mbs: list = field(default_factory=list)
    slice_first_mb: list = field(default_factory=list)
    headers: list = field(default_factory=list)      # the parsed header fields of every slice, in order


# ------------------------------------------------------------------------------------------------ 9.2 residual_block_cavlc
def residual_block(b: Bits, nC: int, maxc: int):
    """Returns (levels of the maxc coefficients in scan order, TotalCoeff)."""
    if nC == -1:
        total, t1 = b.vlc(CDC_TOKEN)
    else:
        total, t1 = b.vlc(COEFF_TOKEN[0 if nC < 2 else 1 if nC < 4 else 2 if nC < 8 else 3])
    coeffs = [0] * maxc
    if total == 0:
        return coeffs, 0
    if total > maxc:
        raise SyntaxError_("TotalCoeff exceeds maxNumCoeff")
    level = []
    suffix_len = 1 if total > 10 and t1 < 3 else 0
    for i in range(total):
        if i < t1:
            level.append(-1 if b.u(1) else 1)
            continue
        prefix = 0
        while b.u(1) == 0:                               # 9.2.2.1 level_prefix
            prefix += 1
        size = 4 if (prefix == 14 and suffix_len == 0) else (prefix - 3 if prefix >= 15 else suffix_len)
        suffix = b.u(size) if size > 0 else 0
        code = (min(15, prefix) << suffix_len) + suffix
        if prefix >= 15 and suffix_len == 0:
            code += 15
        if prefix >= 16:
            code += (1 << (prefix - 3)) - 4096
        if i == t1 and t1 < 3:
            code += 2
        lv = (code + 2) >> 1 if code % 2 == 0 else (-code - 1) >> 1
        level.append(lv)
        if suffix_len == 0:
            suffix_len = 1
        if abs(lv) > (3 << (suffix_len - 1)) and suffix_len < 6:
            suffix_len += 1
    zeros_left = 0
    if total < maxc:
        zeros_left = b.vlc(CDC_TOTAL_ZEROS[total - 1] if nC == -1 else TOTAL_ZEROS[total - 1])
    run = [0] * total
    for i in range(total - 1):
        if zeros_left > 0:
            run[i] = b.vlc(RUN_BEFORE[min(zeros_left, 7) - 1])
            zeros_left -= run[i]
    run[total - 1] = zeros_left
    pos = -1                                             # 9.2.4: highest frequency first
    for i in range(total - 1, -1, -1):
        pos += run[i] + 1
        coeffs[pos] = level[i]
    return coeffs, total


# ------------------------------------------------------------------------------------------------ the picture parser
class _PicState:
    def __init__(self, sps):
        self.sps = sps
        self.mbs = [None] * (sps.mbw * sps.mbh)

    def nb(self, cur: Mb, dx, dy):
        """The macroblock at offset (dx, dy) in macroblocks from `cur`, or None when it is not available (6.4.8: outside the
        picture, not yet decoded or in another slice)."""
        w = self.sps.mbw
        x, y = cur.addr % w + dx, cur.addr // w + dy
        if x < 0 or x >= w or y < 0:
            return None
        n = self.mbs[y * w + x]
        if n is None or n.slice != cur.slice or n.addr >= cur.addr:
            return None
        return n

    def luma_nb(self, cur, bx, by):
        """(macroblock, bx, by) of the 4x4 luma block at (bx, by) in block units relative to `cur` (6.4.11.4)."""
        dx, dy = (bx // 4), (by // 4)
        m = cur if dx == 0 and dy == 0 else self.nb(cur, dx, dy)
        return m, bx % 4, by % 4


def _total_coeff_luma(m, bx, by):
    return int(m.total_coeff[BLK_IDX[(bx, by)]])


def _nc(state, cur, bx, by, chroma=None):
    """9.2.1: nC of the block at (bx, by) (units of 4 samples) of `cur`; chroma = component index for chroma AC."""
    vals = []
    for ox, oy in ((-1, 0), (0, -1)):
        if chroma is None:
            m, x, y = state.luma_nb(cur, bx + ox, by + oy)
        else:
            dx, dy = (bx + ox) // 2, (by + oy) // 2
            m = cur if dx == 0 and dy == 0 else state.nb(cur, dx, dy)
            x, y = (bx + ox) % 2, (by + oy) % 2
        if m is None:
            vals.append(None)
        elif m.kind == "P_Skip":
            vals.append(0)
        elif m.kind == "I_PCM":
            vals.append(16)
        elif chroma is None:
            vals.append(_total_coeff_luma(m, x, y))
        else:
            vals.append(int(m.total_coeff_c[chroma][y * 2 + x]))
    a, b_ = vals
    if a is not None and b_ is not None:
        return (a + b_ + 1) >> 1
    return a if a is not None else (b_ if b_ is not None else 0)


def _i4_pred_mode(state, cur, blk):
    """8.3.1.1: predIntra4x4PredMode of block blk (constrained_intra_pred_flag is 0)."""
    bx, by = BLK_XY[blk]
    modes = []
    for ox, oy in ((-1, 0), (0, -1)):
        m, x, y = state.luma_nb(cur, bx + ox, by + oy)
        if m is None:
            return 2                                     # dcPredModePredictedFlag
        modes.append(m.i4_modes[BLK_IDX[(x, y)]] if m.kind == "I_NxN" else 2)
    return min(modes)


def _mv_neighbours(state, cur):
    """8.4.1.3.2 for a 16x16 partition: (available, refIdx, mv) of A, B, C (C replaced by D when unavailable)."""
    out = []
    a, b_, c = state.nb(cur, -1, 0), state.nb(cur, 0, -1), state.nb(cur, 1, -1)
    if c is None:
        c = state.nb(cur, -1, -1)
    for m in (a, b_, c):
        if m is None:
            out.append((False, -1, (0, 0)))
        elif m.intra:
            out.append((True, -1, (0, 0)))
        else:
            out.append((True, 0, m.mv))
    return out


def mv_pred(state, cur):
    """8.4.1.3: the luma motion vector predictor of a 16x16 partition with refIdxL0 = 0."""
    (avA, rA, mA), (avB, rB, mB), (avC, rC, mC) = _mv_neighbours(state, cur)
    if not avB and not avC and avA:
        rB, mB, rC, mC = rA, mA, rA, mA
    refs = [rA == 0, rB == 0, rC == 0]
    if sum(refs) == 1:
        return (mA, mB, mC)[refs.index(True)]
    return tuple(int(np.median([mA[i], mB[i], mC[i]])) for i in range(2))


def mv_skip(state, cur):
    """8.4.1.1: the P_Skip motion vector."""
    a, b_ = state.nb(cur, -1, 0), state.nb(cur, 0, -1)
    if a is None or b_ is None:
        return (0, 0)
    for m in (a, b_):
        if not m.intra and m.mv == (0, 0):
            return (0, 0)
    return mv_pred(state, cur)


def _residual(b, state, m: Mb, i16: bool):
    """7.3.5.3 residual( 0, 15 ) for ChromaArrayType 1."""
    m.luma = np.zeros((16, 16), np.int64)
    m.total_coeff = np.zeros(16, np.int64)
    m.chroma_dc = np.zeros((2, 4), np.int64)
    m.chroma_ac = np.zeros((2, 4, 16), np.int64)
    m.total_coeff_c = np.zeros((2, 4), np.int64)
    if i16:
        lv, _ = residual_block(b, _nc(state, m, 0, 0), 16)
        m.luma_dc = np.array(lv, np.int64)
    for blk in range(16):
        if not (m.cbp >> (blk >> 2)) & 1:
            continue
        bx, by = BLK_XY[blk]
        nc = _nc(state, m, bx, by)
        if i16:
            lv, tc = residual_block(b, nc, 15)
            m.luma[blk, 1:] = lv
        else:
            lv, tc = residual_block(b, nc, 16)
            m.luma[blk] = lv
        m.total_coeff[blk] = tc
    cc = m.cbp >> 4
    if cc:
        for c in range(2):
            lv, _ = residual_block(b, -1, 4)
            m.chroma_dc[c] = lv
    if cc & 2:
        for c in range(2):
            for blk in range(4):
                lv, tc = residual_block(b, _nc(state, m, blk & 1, blk >> 1, chroma=c), 15)
                m.chroma_ac[c, blk, 1:] = lv
                m.total_coeff_c[c, blk] = tc


def _macroblock_layer(b, state, m: Mb, slice_p: bool, qp: int):
    start = b.pos
    t = b.ue()
    if slice_p:
        if t >= 5:
            t -= 5
        elif t == 0:
            m.kind = "P_L0_16x16"
        else:
            raise SyntaxError_(f"P mb_type {t} is outside the subset")
    if m.kind != "P_L0_16x16":
        if t == 25:
            m.kind = "I_PCM"
        elif t == 0:
            m.kind = "I_NxN"
        elif t <= 24:
            m.kind = "I_16x16"
            m.i16_mode, m.cbp = (t - 1) % 4, ((t - 1) // 4 % 3) << 4 | (15 if t >= 13 else 0)
        else:
            raise SyntaxError_(f"mb_type {t}")
    state.mbs[m.addr] = m
    if m.kind == "I_PCM":
        while not b.byte_aligned():
            if b.u(1):
                raise SyntaxError_("pcm_alignment_zero_bit is 1")
        s = np.array([b.u(8) for _ in range(384)], np.uint8)
        m.pcm = (s[:256].reshape(16, 16), s[256:320].reshape(8, 8), s[320:].reshape(8, 8))
        m.total_coeff = np.full(16, 16, np.int64)
        m.total_coeff_c = np.full((2, 4), 16, np.int64)
        m.qp, m.bits = qp, b.pos - start
        return qp
    if m.kind == "I_NxN":
        m.i4_modes = [0] * 16
        for blk in range(16):
            pm = _i4_pred_mode(state, m, blk)
            if b.u(1):
                m.i4_modes[blk] = pm
            else:
                rem = b.u(3)
                m.i4_modes[blk] = rem if rem < pm else rem + 1
    if m.intra:
        m.chroma_mode = b.ue()
        if m.chroma_mode > 3:
            raise SyntaxError_("intra_chroma_pred_mode")
    else:
        m.mvd = (b.se(), b.se())                         # num_ref_idx_l0_active is 1: no ref_idx_l0
        p = mv_pred(state, m)
        m.mv = (p[0] + m.mvd[0], p[1] + m.mvd[1])
        m.skip_mv = mv_skip(state, m)
    if m.kind != "I_16x16":
        m.cbp = (CBP_INTRA if m.intra else CBP_INTER)[b.ue()]
    if m.cbp or m.kind == "I_16x16":
        qp = (qp + b.se() + 52) % 52                     # 7.4.5 mb_qp_delta
    m.qp = qp
    _residual(b, state, m, m.kind == "I_16x16")
    m.bits = b.pos - start
    return qp


def parse_slice(rbsp: bytes, nal_type: int, nal_ref_idc: int, sps: Sps, pps: dict, state: _PicState, slice_idx: int):
    """7.3.3 slice_header + 7.3.4 slice_data; fills state.mbs.  Returns the header fields."""
    b = Bits(rbsp)
    first_mb, slice_type = b.ue(), b.ue() % 5
    if slice_type not in (0, 2):
        raise SyntaxError_(f"slice_type {slice_type} is outside the subset")
    b.ue()                                               # pic_parameter_set_id
    hdr = dict(first_mb=first_mb, slice_type=slice_type, frame_num=b.u(sps.log2_max_frame_num))
    idr = nal_type == 5
    if idr:
        hdr["idr_pic_id"] = b.ue()
    if sps.poc_type == 0:
        raise SyntaxError_("pic_order_cnt_type 0 is outside the subset")
    if slice_type == 0:
        if b.u(1):                                       # num_ref_idx_active_override_flag
            if b.ue() != 0:
                raise SyntaxError_("more than one reference index")
        if b.u(1):
            raise SyntaxError_("ref_pic_list_modification is outside the subset")
    if nal_ref_idc:
        if idr:
            hdr["no_output_of_prior_pics"], hdr["long_term_reference_flag"] = b.u(1), b.u(1)
        elif b.u(1):
            raise SyntaxError_("adaptive_ref_pic_marking is outside the subset")
    qp = pps["pic_init_qp"] + b.se()
    hdr["qp"] = qp
    if pps["deblocking_filter_control_present_flag"]:
        hdr["disable_deblocking_filter_idc"] = b.ue()
        if hdr["disable_deblocking_filter_idc"] != 1:
            b.se(), b.se()
    slice_p = slice_type == 0
    addr, n = first_mb, sps.mbw * sps.mbh
    more = True
    while more:
        if slice_p:
            run = b.ue()
            for _ in range(run):
                if addr >= n:
                    raise SyntaxError_("mb_skip_run past the end of the picture")
                m = Mb(addr, slice_idx, "P_Skip", qp, total_coeff=np.zeros(16, np.int64), total_coeff_c=np.zeros((2, 4), np.int64))
                state.mbs[addr] = m
                m.mv = mv_skip(state, m)
                addr += 1
            if run:
                more = b.more_rbsp_data()
        if more:
            if addr >= n:
                raise SyntaxError_("macroblock past the end of the picture")
            qp = _macroblock_layer(b, state, Mb(addr, slice_idx, "", qp), slice_p, qp)
            addr += 1
            more = b.more_rbsp_data()
    if b.s[b.pos:] != "1" + "0" * (len(b.s) - b.pos - 1):
        raise SyntaxError_("slice does not end in rbsp_slice_trailing_bits")
    hdr["end_mb"] = addr
    return hdr


class StreamParser:
    """Parses the access units of one stream (one band in striped mode) in decoding order."""

    def __init__(self):
        self.sps = self.pps = None
        self.nal_types = []

    def picture(self, au: bytes) -> Picture:
        pic, state = None, None
        for nal in split_annexb(au):
            if nal[0] & 0x80:
                raise SyntaxError_("forbidden_zero_bit")
            ref_idc, t = nal[0] >> 5 & 3, nal[0] & 31
            self.nal_types.append(t)
            rbsp = unescape(nal)
            if t == 7:
                self.sps = parse_sps(rbsp)
            elif t == 8:
                self.pps = parse_pps(rbsp)
            elif t in (1, 5):
                if state is None:
                    state = _PicState(self.sps)
                hdr = parse_slice(rbsp, t, ref_idc, self.sps, self.pps, state, len(pic.slice_first_mb) if pic else 0)
                if pic is None:
                    pic = Picture(self.sps, t == 5, hdr["frame_num"], hdr["qp"], ref_idc)
                elif hdr["first_mb"] != pic.headers[-1]["end_mb"]:
                    raise SyntaxError_("slices are not contiguous")
                pic.slice_first_mb.append(hdr["first_mb"])
                pic.headers.append(hdr)
            else:
                raise SyntaxError_(f"NAL unit type {t} is outside the subset")
        if pic is None or pic.headers[0]["first_mb"] != 0 or pic.headers[-1]["end_mb"] != len(state.mbs):
            raise SyntaxError_("access unit does not cover the picture")
        pic.mbs = state.mbs
        return pic


def parse_stream(aus):
    p = StreamParser()
    return [p.picture(bytes(a)) for a in aus]
