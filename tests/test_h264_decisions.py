"""The encoder's decisions, macroblock by macroblock, against a second statement of DESIGN.md §5 that shares no code with either
encoder: tests/h264_syntax_refs.py (on tests/h264_syntax.py) parses the bytes and follows the decoded picture buffer,
tests/h264_model.py restates prediction, quantisation, decimation, the intra decision of §5.2, the size rule of §5.7, motion cost, the
lean pass's exits, the search after it (anchor predictor, reduced and exhaustive search, second window, quarter-sample refinement)
and the long-term marking rule.
Byte parity with the oracle and libavcodec's decode pin conformance; these checks pin what is coded.

Per stream (one per band in striped mode) and picture:
  - parser self-check: the model's reconstruction from the parsed syntax equals libavcodec's decode of the same bytes;
  - quantisation: every block's parsed levels equal the model's levels for source − prediction (after decimation in P
    macroblocks), blocks absent from cbp and P_Skip macroblocks included, each inter macroblock predicted from the model's
    reconstruction of the picture its refIdx names;
  - A.3.1: every non-PCM macroblock_layer() is at most 3200 bits, its header within the budget of §5.7, every I_PCM sample equals
    the source, every I_PCM macroblock sized above 3200 bits by the model (intra: M.intra_decide; P: M.p_mb_size at M.decide's
    vector);
  - intra pictures (IDR pictures and scene cuts, §5.2): every macroblock's kind, Intra16x16, chroma and Intra4x4 modes are
    M.intra_decide's, from the model's own reconstruction of its left neighbour;
  - no refIdx-0 P_L0_16x16 macroblock has cbp 0 and its P_Skip vector;
  - motion (§5.3, §5.12, §5.13): every macroblock of a P picture (a scene cut is none) not sent as I_PCM carries exactly the refIdx
    and vector M.decide gives it;
  - the long-term reference (§5.13): the marks, their operations, the override and the picture the DPB names follow the model's
    rule on the model's own changed(k);
  - the SPS: profile, constraint flags, level against Table A-1, reference frames, cropping and the VUI of §5.1.
This file runs them on the oracle's streams; tests/test_h264_decisions_gpu.py on the GPU's."""
from __future__ import annotations

import math
import time

import numpy as np
import pytest

import oracle
from oracle import avdec
from tests import h264_model as M
from tests import h264_syntax_refs as HSR
from tests import layered_scenario as LS
from tests import ltr_content as LC
from tests import ltr_scenario as LTS
from tests import scenario as S
from tests import scut_scenario as SC
from tests import synth
from tests import wide_content as WC
from tests import wide_scenario as WS
from tests.h264_syntax import BLK_XY, Mb, StreamParser, scan_to_raster, split_annexb

MAX_MB_BITS = 3200                       # A.3.1
# Table A-1: level_idc -> MaxFS (macroblocks), levels 3.1 .. 6.2
MAX_FS = {31: 3600, 32: 5120, 40: 8192, 41: 8192, 42: 8704, 50: 22080, 51: 36864, 52: 36864, 60: 139264, 61: 139264, 62: 139264}
# §5.1: the encoders' ladder and its frame-size cap per level — Table A-1's MaxFS, except that 5.1 stops at level 5's 22080 so
# that a 4K picture is 5.2 (whose MaxMBPS carries 4K at 60 fps)
LADDER_CAP = {31: 3600, 42: 8704, 51: 22080, 52: 36864, 62: 139264}


def level_ok(level_idc, mbw, mbh):
    """A.3.1 with Table A-1: the frame size fits MaxFS, and width and height each fit sqrt(8 * MaxFS)."""
    fs = MAX_FS[level_idc]
    bound = math.isqrt(8 * fs)
    return mbw * mbh <= fs and mbw <= bound and mbh <= bound


def smallest_level(mbw, mbh):
    """The level §5.1 names: the first rung of the ladder whose cap holds the frame and that satisfies A.3.1."""
    return next(lv for lv, cap in LADDER_CAP.items() if mbw * mbh <= cap and level_ok(lv, mbw, mbh))


# ------------------------------------------------------------------------------------------------ streams
class Encoded:
    """What one encoder produced for a list of pictures: per band y_start, [(picture index, access unit)], and the source NV12
    (coded size) of every picture."""

    def __init__(self, width, height, cw, ch):
        self.width, self.height, self.cw, self.ch = width, height, cw, ch
        self.bands = {}
        self.sources = []
        self.recon = None                # the encoder's reconstruction after the last picture
        self.flags = 0                   # the session's B2V_FLAG_* word

    @property
    def wide(self):
        return bool(self.flags & WS.FLAG_WIDE_MOTION)

    @property
    def ltr(self):
        return bool(self.flags & LTS.FLAG_LONG_TERM_REF)

    def add(self, index, y_start, au):
        self.bands.setdefault(y_start, []).append((index, au))


def source_nv12(frame, cw, ch):
    h, w = frame.shape[:2]
    y, uv = oracle.csc_nv12(frame, w, h, cw, ch)
    return y, uv[:, 0::2], uv[:, 1::2]


def oracle_side(cfg: S.Config) -> S.OracleSide:
    """The oracle side for cfg.flags: scene cuts (with the long-term reference or not), the long-term reference (wide motion or not),
    wide-range motion (droppable or not), droppable pictures, or none of them."""
    if cfg.flags & SC.FLAG_SCENE_CUT:
        return SC.ScutOracleSide(cfg)
    if cfg.flags & LTS.FLAG_LONG_TERM_REF:
        return LTS.LtrOracleSide(cfg)
    if cfg.flags & WS.FLAG_WIDE_MOTION:
        return WS.WideOracleSide(cfg)
    return LS.LayeredOracleSide(cfg) if cfg.flags & LS.FLAG_DROPPABLE else S.OracleSide(cfg)


def encode_oracle(cfg: S.Config, frames, idr_at=(0,), qps=None, each=None) -> Encoded:
    """The oracle encoder over `frames` (IDR at the indices in idr_at, QP per picture from qps when given); each(i, encoder, bands)
    after picture i when given."""
    side = oracle_side(cfg)
    enc = side.enc
    out = Encoded(cfg.width, cfg.height, enc.cw, enc.ch)
    out.flags = cfg.flags
    for i, f in enumerate(frames):
        if i in idr_at:
            side.control(S.request_idr())
        if qps is not None:
            side.control(S.set_qp(qps[i]))
        x = side.picture(f, "")
        out.sources.append(source_nv12(f, enc.cw, enc.ch))
        for y0, au in x.bands:
            out.add(i, y0, au)
        if each is not None:
            each(i, enc, x.bands)
    out.recon = enc.recon()
    return out


# ------------------------------------------------------------------------------------------------ the checks
class Stats:
    def __init__(self):
        self.kinds = {}
        self.max_bits = 0
        self.pictures = 0
        self.levels = []                  # SPS level_idc seen
        self.last = {}                    # band y_start -> the model's last reconstruction (Y, U, V)
        self.exits = {}                   # lean-pass class (and "predictor lean" / "predictor search" / "long-term over predictor") -> count
        self.marks = []                   # (band y_start, decoding index) of the pictures that mark a long-term picture
        self.mmco1_wrap = 0               # marking pictures whose MMCO 1 names a frame across the frame_num wrap
        self.mark_at_fn0 = 0              # marking pictures with frame_num 0 (MMCO 3 names PicNum -1)
        self.lt_age = 0                   # the largest distance (pictures) from a long-term picture to a picture predicting from it
        self.lt_fn_twin = 0               # refIdx-1 macroblocks in pictures whose short-term reference has the long-term frame_num
        self.skip_next_to_lt = 0          # refIdx-0 P_Skip macroblocks with a refIdx-1 neighbour left or above
        self.scaled = 0                   # predictor-class macroblocks of pictures whose reference distances differ, previous vector fractional
        self.pcm_two_refs = 0             # I_PCM macroblocks in pictures with two references
        self.paths = {}                   # how M.decide found vectors ("refined search", "anchor predictor", ...) -> count
        # the intra decision (§5.2) and the I_PCM rule (§5.7), from the model where the stream carries what it decides
        self.i4_row0, self.i4_rows = set(), set()     # Intra4x4 modes of I_NxN macroblocks in block row 0 / rows 1..3
        self.i16_modes, self.chroma_modes = set(), set()
        self.i4_untried = 0               # intra macroblocks whose Intra16x16 SAD kept the gate of 32·λ shut
        self.gate_decides = 0             # ... where Intra4x4 would have won the comparison
        self.compared = {}                # kind kept where Intra4x4 was tried ("I_NxN" / "I_16x16") -> count
        self.ties = {}                    # SAD ties the mode index resolved: "I16 H over DC", "chroma DC over H" -> count
        self.slice_starts = 0             # intra macroblocks that start a slice inside a row (no left neighbour)
        self.min_dj = None                # the smallest |J4 − J16| where Intra4x4 was tried
        self.max_coded = {"I": 0, "P": 0}           # the largest §5.7 size of a coded macroblock, intra / inter
        self.min_pcm = {"I": None, "P": None}       # the smallest model size of an I_PCM macroblock, in intra / P pictures
        self.cut_pictures = 0             # non-IDR pictures of I slices (scene cuts)
        self.cut_pcm = 0                  # I_PCM macroblocks in them

    def count(self, kind, d=None):
        d = self.kinds if d is None else d
        d[kind] = d.get(kind, 0) + 1

    def pcm_size(self, pic_type, size):
        self.min_pcm[pic_type] = size if self.min_pcm[pic_type] is None else min(self.min_pcm[pic_type], size)


def check_sps(sps, width, height, y_start, band_h, mbw, mbh_band, stats, flags=0):
    """§5.1 (and §5.13 with B2V_FLAG_LONG_TERM_REF: two reference frames, two frames of decoded picture buffer)."""
    stats.levels.append(sps.level_idc)
    refs = 2 if flags & LTS.FLAG_LONG_TERM_REF else 1
    assert sps.profile_idc == 66 and sps.constraint_flags & 0xC0 == 0xC0, "Constrained Baseline (set0 | set1)"
    assert (sps.mbw, sps.mbh) == (mbw, mbh_band)
    assert sps.width == width and sps.height == band_h, (sps.width, sps.height, width, band_h, y_start)
    assert sps.crop[0] == 0 and sps.crop[2] == 0
    assert sps.poc_type == 2 and sps.max_num_ref_frames == refs
    assert level_ok(sps.level_idc, sps.mbw, sps.mbh), f"level_idc {sps.level_idc} does not hold {sps.mbw}x{sps.mbh} macroblocks"
    assert sps.level_idc == smallest_level(sps.mbw, sps.mbh)
    v = sps.vui
    assert (v.get("video_format"), v.get("video_full_range_flag")) == (5, 0)
    assert (v.get("colour_primaries"), v.get("transfer_characteristics"), v.get("matrix_coefficients")) == (1, 1, 1)
    assert (v.get("chroma_sample_loc_type_top"), v.get("chroma_sample_loc_type_bottom")) == (1, 1)
    assert (v.get("max_num_reorder_frames"), v.get("max_dec_frame_buffering")) == (0, refs)
    assert v["timing_info_present_flag"] == 0 and v["nal_hrd"] == 0 and v["vcl_hrd"] == 0


def _avail(pic, addr, mbw):
    """Neighbour availability (A, B, C, D) of macroblock addr: inside the picture and in the same slice."""
    x, y = addr % mbw, addr // mbw
    s = pic.mbs[addr].slice

    def ok(dx, dy):
        nx, ny = x + dx, y + dy
        return 0 <= nx < mbw and ny >= 0 and pic.mbs[ny * mbw + nx].slice == s
    return M.Avail(ok(-1, 0), ok(0, -1), ok(1, -1), ok(-1, -1))


def check_picture(pic, recs, src, where, stats, wide=False):
    """Reconstructs `pic` from its syntax with the model (recs: the model's reconstructions of this stream by decoding index; an
    inter macroblock predicts from recs[m.ref_pic], the picture its refIdx names) and checks every macroblock's levels against the
    model's levels for the source `src` (Y, U, V of the stream's coded size), and that every macroblock sent coded fits the I_PCM
    rule's budget, its header included (wide: a wide-motion stream).  Returns the reconstruction (Y, U, V)."""
    mbw, mbh = pic.sps.mbw, pic.sps.mbh
    rec = [np.zeros((mbh * 16, mbw * 16), np.uint8), np.zeros((mbh * 8, mbw * 8), np.uint8), np.zeros((mbh * 8, mbw * 8), np.uint8)]
    sy, su, sv = (p.astype(np.int64) for p in src)
    for m in pic.mbs:
        mbx, mby = m.addr % mbw, m.addr // mbw
        x0, y0, xc, yc = 16 * mbx, 16 * mby, 8 * mbx, 8 * mby
        at = f"{where} mb ({mbx},{mby}) {m.kind} qp {m.qp}"
        stats.count(m.kind)
        if m.kind == "I_PCM":
            rec[0][y0:y0 + 16, x0:x0 + 16], rec[1][yc:yc + 8, xc:xc + 8], rec[2][yc:yc + 8, xc:xc + 8] = m.pcm
            for k, (s_, p) in enumerate(zip((sy[y0:y0 + 16, x0:x0 + 16], su[yc:yc + 8, xc:xc + 8], sv[yc:yc + 8, xc:xc + 8]), m.pcm)):
                assert np.array_equal(s_, p), f"{at}: I_PCM samples of plane {k} differ from the source"
            continue
        if m.kind != "P_Skip":
            assert m.bits <= MAX_MB_BITS, f"{at}: macroblock_layer() of {m.bits} bits (A.3.1 limit 3200)"
            budget = M.header_budget(m, wide)
            assert m.header_bits <= budget, f"{at}: a header of {m.header_bits} bits (ref_idx {m.ref_idx}, mvd {m.mvd}), budget {budget}"
            est = M.mb_size_estimate(m, wide)
            assert m.bits <= est, f"{at}: {m.bits} bits coded, more than the {est} of the size rule"     # the rule only overstates
            assert est <= MAX_MB_BITS, f"{at}: sized {est} bits by the rule of §5.7 (wide {wide}), coded instead of I_PCM"
            stats.max_bits = max(stats.max_bits, m.bits)
            t = "I" if m.intra else "P"
            stats.max_coded[t] = max(stats.max_coded[t], est)
        if m.kind == "P_L0_16x16" and m.ref_idx == 0:
            assert not (m.cbp == 0 and m.mv == m.skip_mv), f"{at}: cbp 0 and the P_Skip vector {m.mv}, coded as P_L0_16x16"
        qp, intra = m.qp, m.intra
        av = _avail(pic, m.addr, mbw)
        sblk = sy[y0:y0 + 16, x0:x0 + 16]
        ref = None if intra else recs[m.ref_pic]
        # ---- luma
        if m.kind == "I_NxN":
            for blk in range(16):
                bx, by = BLK_XY[blk]
                P = M.intra4x4_neighbours(rec[0], mbx, mby, blk, av)
                pred = M.intra4x4_pred(m.i4_modes[blk], P)
                r = slice(4 * by, 4 * by + 4), slice(4 * bx, 4 * bx + 4)
                lv, _ = M.quant_block(sblk[r] - pred, qp, True)
                assert np.array_equal(M.raster_to_scan(lv), m.luma[blk]), f"{at}: Intra4x4 block {blk} levels {m.luma[blk]} != model {M.raster_to_scan(lv)}"
                res = M.inverse4x4(M.dequant4x4(m.luma_raster(blk), qp))
                rec[0][y0 + 4 * by:y0 + 4 * by + 4, x0 + 4 * bx:x0 + 4 * bx + 4] = M.clip1(pred + res)
        else:
            if m.kind == "I_16x16":
                pred = M.intra16_pred(m.i16_mode, *M.mb_edges(rec[0], x0, y0, 16, av))
            else:
                pred = M.luma_inter(ref[0], x0, y0, m.mv)
            model = np.zeros((16, 16), np.int64)
            w_dc = np.zeros((4, 4), np.int64)
            for blk in range(16):
                bx, by = BLK_XY[blk]
                r = slice(4 * by, 4 * by + 4), slice(4 * bx, 4 * bx + 4)
                lv, w = M.quant_block(sblk[r] - pred[r], qp, intra, with_dc=not intra)
                model[blk], w_dc[by, bx] = M.raster_to_scan(lv), w[0, 0]
            parsed = m.luma if m.luma is not None else np.zeros((16, 16), np.int64)
            if intra:
                dc = M.i16_dc_levels(w_dc, qp)
                assert np.array_equal(M.raster_to_scan(dc), m.luma_dc), f"{at}: Intra16x16 DC levels {m.luma_dc} != model {M.raster_to_scan(dc)}"
                dcy = M.luma_dc_dequant(scan_to_raster(m.luma_dc), qp)
            else:
                model = M.decimate_levels(model)
            for blk in range(16):
                assert np.array_equal(model[blk], parsed[blk]), f"{at}: luma block {blk} levels {parsed[blk]} != model {model[blk]}"
            for blk in range(16):
                bx, by = BLK_XY[blk]
                d = M.dequant4x4(scan_to_raster(parsed[blk]), qp)
                if intra:
                    d[0, 0] = dcy[by, bx]
                r = slice(4 * by, 4 * by + 4), slice(4 * bx, 4 * bx + 4)
                rec[0][y0 + 4 * by:y0 + 4 * by + 4, x0 + 4 * bx:x0 + 4 * bx + 4] = M.clip1(pred[r] + M.inverse4x4(d))
        # ---- chroma
        qpc = M.QPC[qp]
        for c, sc in ((0, su), (1, sv)):
            if intra:
                pc = M.chroma_pred(m.chroma_mode, *M.mb_edges(rec[1 + c], xc, yc, 8, av))
            else:
                pc = M.chroma_inter(ref[1 + c], xc, yc, m.mv)
            scb = sc[yc:yc + 8, xc:xc + 8]
            w_dc = np.zeros((2, 2), np.int64)
            ac = np.zeros((4, 16), np.int64)
            for blk in range(4):
                bx, by = blk & 1, blk >> 1
                r = slice(4 * by, 4 * by + 4), slice(4 * bx, 4 * bx + 4)
                lv, w = M.quant_block(scb[r] - pc[r], qpc, intra, with_dc=False)
                ac[blk], w_dc[by, bx] = M.raster_to_scan(lv), w[0, 0]
            dc = M.chroma_dc_levels(w_dc, qpc, intra).reshape(4)
            p_dc = m.chroma_dc[c] if m.chroma_dc is not None else np.zeros(4, np.int64)
            p_ac = m.chroma_ac[c] if m.chroma_ac is not None else np.zeros((4, 16), np.int64)
            assert np.array_equal(dc, p_dc), f"{at}: chroma {c} DC levels {p_dc} != model {dc}"
            assert np.array_equal(ac, p_ac), f"{at}: chroma {c} AC levels {p_ac.tolist()} != model {ac.tolist()}"
            dcc = M.chroma_dc_dequant(p_dc.reshape(2, 2), qpc)
            for blk in range(4):
                bx, by = blk & 1, blk >> 1
                d = M.dequant4x4(scan_to_raster(p_ac[blk]), qpc)
                d[0, 0] = dcc[by, bx]
                r = slice(4 * by, 4 * by + 4), slice(4 * bx, 4 * bx + 4)
                rec[1 + c][yc + 4 * by:yc + 4 * by + 4, xc + 4 * bx:xc + 4 * bx + 4] = M.clip1(pc[r] + M.inverse4x4(d))
    return rec


def is_intra_picture(pic):
    """An IDR picture or a scene cut (§5.14): every slice an I slice."""
    return all(h["slice_type"] == 2 for h in pic.headers)


def check_intra(pic, src, rec, where, stats):
    """§5.2 on intra picture `pic` (an IDR picture or a scene cut): its slices never span rows, and every macroblock carries the kind
    and the modes M.intra_picture decides from the source `src` (Y, U, V) on the model's own reconstruction, which must equal `rec`,
    the reconstruction check_picture made from the parsed syntax.  A coded macroblock's model size is its size by the rule of §5.7;
    an I_PCM one's exceeds 3200 bits."""
    mbw, mbh = pic.sps.mbw, pic.sps.mbh
    slice_of = [m.slice for m in pic.mbs]
    for m in pic.mbs:
        assert m.qp == pic.qp, f"{where}: mb {m.addr} at QP {m.qp} in a picture of QP {pic.qp}"
        assert m.addr < mbw or slice_of[m.addr - mbw] != m.slice, f"{where}: the slice of mb {m.addr} spans rows"
    decided, mrec = M.intra_picture(src, slice_of, mbw, mbh, pic.qp)
    for m in pic.mbs:
        r, i = decided[m.addr]
        mbx, mby = m.addr % mbw, m.addr // mbw
        at = f"{where} mb ({mbx},{mby}) {m.kind} qp {m.qp}"
        why = f"model: {r.kind[i]}, size {r.size[i]}, Intra4x4 tried {r.tried[i]}, J16 {r.j16[i]}, J4 {r.j4[i]}"
        assert m.kind == r.kind[i], f"{at}: {why}"
        if m.kind == "I_PCM":
            assert r.size[i] > M.MB_BITS_LIMIT
            stats.pcm_size("I", int(r.size[i]))
            stats.cut_pcm += not pic.idr
        else:
            assert r.size[i] == M.mb_size_estimate(m), f"{at}: size {M.mb_size_estimate(m)} by the parsed levels, {why}"
            assert m.chroma_mode == r.chroma_mode[i], f"{at}: chroma mode {m.chroma_mode}, the model's {r.chroma_mode[i]}"
            stats.chroma_modes.add(m.chroma_mode)
            if r.chroma_tie[i]:
                stats.count("chroma DC over H", stats.ties)
            if m.kind == "I_16x16":
                assert m.i16_mode == r.i16_mode[i], f"{at}: Intra16x16 mode {m.i16_mode}, the model's {r.i16_mode[i]} ({why})"
                stats.i16_modes.add(m.i16_mode)
                if r.i16_tie[i]:
                    stats.count("I16 H over DC", stats.ties)
            else:
                assert list(m.i4_modes) == list(r.i4_modes[i]), f"{at}: Intra4x4 modes {m.i4_modes}, the model's {r.i4_modes[i].tolist()}"
                for blk, mode in enumerate(m.i4_modes):
                    (stats.i4_rows if BLK_XY[blk][1] else stats.i4_row0).add(mode)
            if r.tried[i]:
                stats.count(m.kind, stats.compared)
                dj = abs(int(r.j4[i]) - int(r.j16[i]))
                stats.min_dj = dj if stats.min_dj is None else min(stats.min_dj, dj)
        stats.i4_untried += not r.tried[i]
        stats.gate_decides += not r.tried[i] and m.kind != "I_PCM" and r.j4[i] < r.j16[i]
        stats.slice_starts += mbx > 0 and slice_of[m.addr - 1] != m.slice
    for c in range(3):
        assert np.array_equal(mrec[c], rec[c]), f"{where}: the model's reconstruction of plane {c} != the parsed one"


def check_exits(pic, prev, recs, src, where, stats, wide=False, dec=None):
    """Every macroblock of P picture `pic` against the model's decision (M.decide) from the source `src` (Y, U, V), the model's
    reconstructions of refIdx 0 and of the long-term picture (refIdx 1, while the picture has two references), the previous
    picture's parsed records `prev` (the picture just before in decoding order, reference or not) and, with wide motion, dec: the
    decimated luma of this picture's source and of its reference's.  Anchors are decided first, then the rest with their anchor's
    decision.  Every macroblock not sent as I_PCM must carry exactly the model's refIdx and vector (P_Skip: its inferred vector); every
    I_PCM one must be sized above 3200 bits by the model at that vector (M.p_mb_size)."""
    mbw, mbh = pic.sps.mbw, pic.sps.mbh
    ref = recs[pic.ref_list[0]][0]
    lt = recs[pic.ref_list[1]][0] if len(pic.ref_list) > 1 else None
    dist = (pic.index - pic.ref_list[0], prev.index - prev.ref_list[0] if prev.ref_list else 1)
    y = src[0].astype(np.int64)
    anchor = {m.addr: M.anchor_of(m.addr % mbw, m.addr // mbw, mbw, 0, mbh) for m in pic.mbs}
    decided = {}
    for m in sorted(pic.mbs, key=lambda m: anchor[m.addr] != (m.addr % mbw, m.addr // mbw)):       # anchors first
        mbx, mby = m.addr % mbw, m.addr // mbw
        x0, y0 = 16 * mbx, 16 * mby
        pm = prev.mbs[m.addr]
        blk = y[y0:y0 + 16, x0:x0 + 16]
        is_anchor = anchor[m.addr] == (mbx, mby)
        coarse = None
        if wide and is_anchor:
            coarse = M.coarse_search(dec[0], dec[1], mbx, mby, mbw, 0, mbh, M.sad(blk, ref[y0:y0 + 16, x0:x0 + 16]), pic.qp)
        d = M.decide(blk, ref, lt, pm, x0, y0, pic.qp, wide, dist, None if is_anchor else decided[anchor[m.addr]], coarse)
        decided[(mbx, mby)] = d
        ex = d.ex
        if m.kind == "I_PCM":
            size = M.p_mb_size([p[k * y0 // 16:k * (y0 + 16) // 16, k * x0 // 16:k * (x0 + 16) // 16] for p, k in zip(src, (16, 8, 8))],
                               recs[pic.ref_list[d.ref_idx]], x0, y0, d.mv, pic.qp, wide)
            assert size > M.MB_BITS_LIMIT, f"{where} mb ({mbx},{mby}): I_PCM, sized {size} bits at refIdx {d.ref_idx} mv {d.mv}"
            stats.pcm_size("P", size)
        else:
            assert (m.ref_idx, m.mv) == (d.ref_idx, d.mv), \
                f"{where} mb ({mbx},{mby}): the model decides refIdx {d.ref_idx} mv {d.mv} ({d.path}, class {ex.cls}, k {ex.k}, " \
                f"refined {d.refined}, second window {d.second}) but coded {m.kind} refIdx {m.ref_idx} mv {m.mv}"
        stats.count(ex.cls, stats.exits)
        if ex.cls == "predictor":
            stats.count("predictor lean" if ex.lean else "predictor search", stats.exits)
            if dist[0] != dist[1] and (pm.mv[0] | pm.mv[1]) & 3:
                stats.scaled += 1
                # the candidate halving toward zero would give: where it differs, only the rounding of §5.12 codes this vector
                toward = M.predictor_candidate(tuple(int(c / 2) for c in pm.mv), wide) if dist[0] < dist[1] else None
                if toward is not None and toward[0] != ex.k:
                    stats.count("scaled rounding decides", stats.paths)
        if ex.cls == "long-term" and ex.search_pred:
            inside = 16 <= x0 and x0 + 32 <= ref.shape[1]
            stats.count("long-term over edge predictor" if not inside else "long-term over fractional predictor", stats.exits)
        d13 = max(abs(d.full[0] - d.centre[0]), abs(d.full[1] - d.centre[1])) == 13
        for name, on in (("refined search", d.path == "search" and d.refined),
                         ("refined predictor", d.path == "predictor" and d.refined),
                         ("anchor predictor", d.path == "anchor predictor"),
                         ("reduced search", d.path == "reduced search"),
                         ("second window", d.second),
                         # where a mistake in one rule changes the vector: each names the rule it exposes
                         ("refined at |d| = 13", d.refined and d13),
                         ("refined with SAD >= 4096", d.refined and d.sad >= 4096),
                         ("reduced search at |dy| = 2", d.path == "reduced search" and abs(d.full[1]) == 2),
                         ("anchor candidate rounded up", d.path == "anchor predictor" and d.full != (d.src[0] >> 2, d.src[1] >> 2)),
                         ("refinement moves an inside fractional hit", d.path == "predictor" and d.refined and d.mv != (4 * d.full[0], 4 * d.full[1])
                          and x0 - 16 + d.centre[0] >= 0 and x0 + 32 + d.centre[0] <= ref.shape[1])):
            if on:
                stats.count(name, stats.paths)
        if m.ref_idx == 1 and pic.ref_frame_nums[0] == pic.ref_frame_nums[1]:
            stats.lt_fn_twin += 1
        stats.pcm_two_refs += m.kind == "I_PCM" and lt is not None
        if m.kind == "P_Skip" and lt is not None:
            if (mbx > 0 and pic.mbs[m.addr - 1].ref_idx == 1) or (mby > 0 and pic.mbs[m.addr - mbw].ref_idx == 1):
                stats.skip_next_to_lt += 1


class LtrModel:
    """The long-term reference of §5.13 restated on one stream: the model's changed(k) from the source and the model's reconstruction
    of picture k − 1, the marking rule, whether a long-term picture exists and which."""

    def __init__(self, mbs):
        self.mbs, self.prev_changed, self.lt = mbs, mbs, None

    def picture(self, pic, recs, src_y, stats, y_start):
        """Checks picture `pic`'s marking, operations, override and long-term reference against the rule, then advances."""
        where = f"picture {pic.index} band {y_start}"
        if pic.idr:
            assert all("mmco" not in h and not h.get("long_term_reference_flag") for h in pic.headers), where
            self.prev_changed, self.lt = self.mbs, None
            return
        changed = M.changed_count(src_y, recs[pic.index - 1][0], pic.qp)
        mark = M.marks(changed, self.prev_changed, self.mbs)
        cut = is_intra_picture(pic)      # a scene cut keeps its P picture's marking; its I slices carry no override
        for h in pic.headers:
            assert h.get("mmco") == (M.marking_ops(self.lt is not None) if mark else None), \
                f"{where}: operations {h.get('mmco')}, the rule says mark {mark} (changed {changed}, before {self.prev_changed})"
            if not cut:
                assert h.get("num_ref_idx_active", 1) == (2 if self.lt is not None else 1), f"{where}: override {h.get('num_ref_idx_active')}"
        if not cut:
            assert pic.ref_list == ([pic.index - 1] + ([self.lt] if self.lt is not None else [])), (where, pic.ref_list, self.lt)
        if self.lt is not None:
            stats.lt_age = max(stats.lt_age, pic.index - self.lt)
        if mark:
            stats.marks.append((y_start, pic.index))
            stats.mark_at_fn0 += pic.frame_num == 0
            if self.lt is None:
                stats.mmco1_wrap += pic.frame_num < 2
            self.lt = pic.index - 1
        assert pic.long_term == ([self.lt] if self.lt is not None else []), (where, pic.long_term, self.lt)
        self.prev_changed = changed


def check_encoded(e: Encoded, stripe_rows=0):
    """All per-picture checks over every band stream of `e`; returns Stats.  The reader's DPB names the picture each inter
    macroblock predicts from; the model keeps its reconstructions by decoding index."""
    stats = Stats()
    mbw, mbh = e.cw // 16, e.ch // 16
    for y_start, items in sorted(e.bands.items()):
        band_mbh = min(mbh - y_start // 16, stripe_rows or mbh)
        band_h = min(e.height - y_start, band_mbh * 16)
        pics = HSR.parse_stream([au for _, au in items])
        decoded = avdec.decode_stream([au for _, au in items], quiet=True)
        assert len(decoded) == len(pics)
        recs, ltr = [], LtrModel(mbw * band_mbh) if e.ltr else None
        for k, ((index, _), pic, dec) in enumerate(zip(items, pics, decoded)):
            where = f"picture {index} band {y_start}"
            if pic.idr:
                check_sps(pic.sps, e.width, e.height, y_start, band_h, mbw, band_mbh, stats, e.flags)
            assert pic.sps.mbh == band_mbh
            src = [p[y_start // k_: y_start // k_ + band_mbh * 16 // k_] for p, k_ in zip(e.sources[index], (1, 2, 2))]
            pic.ref_frame_nums = [pics[i].frame_num for i in pic.ref_list]
            rec = check_picture(pic, recs, src, where, stats, e.wide)
            intra = is_intra_picture(pic)
            if intra:
                check_intra(pic, src, rec, where, stats)
                stats.cut_pictures += not pic.idr
            vh, vw = pic.sps.height, pic.sps.width
            for c, (r, d) in enumerate(zip(rec, dec)):
                s = 1 if c == 0 else 2
                assert np.array_equal(r[: vh // s, : vw // s], d), f"{where}: model reconstruction of plane {c} != libavcodec's decode"
            # the exits need the previous picture's records: a band left unsent (all skipped) in between hides them
            if not intra and k > 0 and items[k - 1][0] == index - 1:
                dec = None
                if e.wide:     # the coarse search's planes: the decimated sources of this picture and of its reference
                    ref_src = e.sources[items[pic.ref_list[0]][0]][0][y_start:y_start + band_mbh * 16]
                    dec = M.decimate(src[0]), M.decimate(ref_src)
                check_exits(pic, pics[k - 1], recs, src, where, stats, e.wide, dec)
            if ltr is not None:
                ltr.picture(pic, recs, src[0], stats, y_start)
            recs.append(rec)
            stats.pictures += 1
        stats.last[y_start] = rec
    return stats


def check_recon(e: Encoded, stats):
    """The model's last reconstruction of every band equals the encoder's own reconstruction buffer."""
    ry, ruv = e.recon
    for y_start, (y, u, v) in stats.last.items():
        n = y.shape[0]
        assert np.array_equal(ry[y_start:y_start + n], y)
        assert np.array_equal(ruv[y_start // 2:(y_start + n) // 2, 0::2], u)
        assert np.array_equal(ruv[y_start // 2:(y_start + n) // 2, 1::2], v)


# ------------------------------------------------------------------------------------------------ configurations
def grey(w, h, luma_of_grey, y):
    """BGRA picture whose oracle CSC gives exactly the luma plane y (values 16..235) and chroma 128."""
    g = luma_of_grey[np.asarray(y, np.int64)]
    f = np.empty((h, w, 4), np.uint8)
    f[..., 0] = f[..., 1] = f[..., 2] = g
    f[..., 3] = 255
    return f


def grey_table():
    """Grey value per luma value 16..235 (oracle CSC of BGRA grey)."""
    ramp = np.zeros((16, 256, 4), np.uint8)
    ramp[..., :3] = np.arange(256, dtype=np.uint8)[None, :, None]
    ramp[..., 3] = 255
    y, uv = oracle.csc_nv12(ramp)
    inv = np.full(256, -1, np.int64)
    for g in range(256):
        inv[y[0, g]] = g if inv[y[0, g]] < 0 else inv[y[0, g]]
    assert (inv[16:236] >= 0).all() and (uv == 128).all()
    return inv


def cases():
    """(id, Config, frames, idr_at, qps, stripe_rows): the configurations of both test files."""
    out = []
    for qp in (0, 10, 26, 40, 51):
        w, h = (48, 32) if qp < 20 else (160, 96)
        fr = [synth.desktop(w, h, t) for t in range(3)] if qp >= 20 else [synth.noise(w, h, 3), synth.noise(w, h, 3), synth.desktop(w, h, 0)]
        out.append((f"qp{qp}", S.Config(w, h, qp=qp), fr, (0,), None, 0))
    out.append(("pcm_noise_qp0_4", S.Config(64, 48, qp=0), [synth.noise(64, 48, s) for s in (5, 6, 7)], (0,), [0, 2, 4], 0))
    out.append(("cbr_mid_idr", S.Config(160, 96, rc_mode=S.CBR, kbps=400, fps=30.0), [synth.desktop(160, 96, t) for t in range(6)], (0, 3), None, 0))
    out.append(("idr_subrow_p_rows1", S.Config(320, 64, qp=30, slice_rows=1, idr_slice_mbs=7), [synth.desktop(320, 64, t) for t in range(3)], (0,), None, 0))
    out.append(("p_rows8", S.Config(160, 160, qp=28, slice_rows=8), [synth.desktop(160, 160, t) for t in range(3)], (0,), None, 0))
    out.append(("p_whole", S.Config(160, 96, qp=28, slice_rows=100), [synth.desktop(160, 96, t) for t in range(3)], (0,), None, 0))
    out.append(("striped", S.Config(192, 112, qp=27, slice_rows=1, stripe_rows=3), [synth.desktop(192, 112, t) for t in range(3)], (0,), None, 3))
    out.append(("crop_130x70", S.Config(130, 70, qp=24), [synth.gradient(130, 70, t) for t in range(3)], (0,), None, 0))
    out.append(("one_mb", S.Config(16, 16, qp=20), [synth.noise(16, 16, 4), synth.noise(16, 16, 5)], (0,), None, 0))
    out.append(("predictor_paths", S.Config(130, 70, qp=30), synth.predictor_paths(130, 70), (0,), None, 0))
    still = synth.desktop(96, 64, 0)
    out.append(("paintover_burst", S.Config(96, 64, qp=40, paint=(2, 20, 3)), [still] * 8, (0,), None, 0))
    return out + wide_cases() + ltr_cases() + motion_cases() + intra_cases()


WIDE = WS.FLAG_WIDE_MOTION
LTR = LTS.FLAG_LONG_TERM_REF


def blocky_noise(w, h, x0, y0, seed=11):
    """The window at (x0, y0) of one large plane of 2x2-blocky mid-range grey noise, as a BGRA picture."""
    rng = np.random.default_rng(seed)
    luma = rng.integers(48, 208, (h // 2 + 160, w // 2 + 160)).repeat(2, 0).repeat(2, 1)
    return grey(w, h, grey_table(), luma[y0:y0 + h, x0:x0 + w])


def band_bottom_scroll(w, h, rows, sx=0, seed=13):
    """Two BGRA pictures of 2x2-blocky grey noise, the second scrolled up by 4 px and left by sx px, with the last 4 luma rows of every
    band of `rows` macroblock rows dark in the second (4 rows lower in the first, the first 4 of the next band): the bottom group of
    each band matches the reference exactly one decimated row below the band, where the coarse search must not look."""
    rng = np.random.default_rng(seed)
    luma = rng.integers(48, 208, ((h + 4) // 2 + 1, (w + sx) // 2 + 1)).repeat(2, 0).repeat(2, 1)[:h + 4, :w + sx]
    for y in range(16 * rows, h, 16 * rows):
        luma[y:y + 4] = 16
    inv = grey_table()
    return [grey(w, h, inv, luma[:h, :w]), grey(w, h, inv, luma[4:4 + h, sx:sx + w])]


def moving_noise(w, h, n, v, seed=3):
    """n BGRA pictures of 2x2-blocky grey noise moving by v px per picture (content at (x, y) was at (x, y) + v one picture earlier:
    true vector v) with fresh noise on top, its amplitude rising from 0 at the left edge to 64 at the right edge: residuals from
    none to beyond the limit of A.3.1."""
    rng = np.random.default_rng(seed)
    pw, ph = w + abs(v[0]) * n, h + abs(v[1]) * n
    base = rng.integers(40, 216, (ph // 2 + 1, pw // 2 + 1)).repeat(2, 0).repeat(2, 1)
    inv = grey_table()
    amp = np.linspace(0, 64, w)[None, :]
    out = []
    for t in range(n):
        x0, y0 = (t * c + (n - 1) * max(0, -c) for c in v)
        fresh = np.rint(amp * rng.uniform(-1, 1, (h, w))).astype(np.int64)
        out.append(grey(w, h, inv, np.clip(base[y0:y0 + h, x0:x0 + w] + fresh, 16, 235)))
    return out


def wide_cases():
    """Wide-range motion (B2V_FLAG_WIDE_MOTION, §5.3): the configurations of both files with the flag on."""
    out = [("wide_scroll40", S.Config(640, 368, qp=26, flags=WIDE), [WC.desktop_scroll(640, 368, t, 40) for t in range(3)], (0,), None, 0),
           ("wide_scroll250_tall", S.Config(96, 640, qp=26, flags=WIDE), [WC.desktop_scroll(96, 640, t, 250) for t in range(3)], (0,), None, 0),
           # mbw = 21: a group of one macroblock column at the right edge; the window leaves through the top-left corner
           ("wide_drag_corner", S.Config(336, 208, qp=26, flags=WIDE),
            [WC.drag(336, 208, t, (-37, -29), (150, 100), 160, 112) for t in range(6)], (0,), None, 0),
           # bands of 3 macroblock rows (and one of 2): every group is partial, the coarse search stops at each band's edges
           ("wide_drag_striped3", S.Config(320, 176, qp=27, slice_rows=1, stripe_rows=3, flags=WIDE),
            [WC.drag(320, 176, t, (-70, 6), (220, 30), 96, 112) for t in range(3)], (0,), None, 3),
           # droppable: pictures 1 and 3 are non-reference, pictures 2 and 4 predict from two back (256 px, beyond the range)
           ("wide_scroll128_droppable", S.Config(160, 480, qp=26, flags=WIDE | LS.FLAG_DROPPABLE),
            [WC.desktop_scroll(160, 480, t, 128) for t in range(5)], (0,), None, 0),
           ("wide_pcm_noise_qp0_4", S.Config(224, 128, qp=0, flags=WIDE), moving_noise(224, 128, 3, (-100, 60)), (0,), [0, 2, 4], 0)]
    return out


def waves(w, h, t, parts, amp=40):
    """BGRA picture t of grey content whose rows [y0, y1) hold a vertical-bar cosine of `period` px moving left by `step` px per
    picture, for (y0, y1, period, step) in parts (exact at every t: a step of half a period repeats the content two pictures on)."""
    inv = grey_table()
    x = np.arange(w)[None, :]
    luma = np.full((h, w), 128.0)
    for y0, y1, period, step in parts:
        luma[y0:y1] = 128 + amp * np.cos(2 * np.pi * (x + step * t) / period)
    return grey(w, h, inv, np.rint(luma).astype(np.int64))


def wrap_content(w, h):
    """513 pictures of flat grey for frame_num's wrap (8 bits): content A still for pictures 0..255, B from 256 on (picture 256 marks picture 255,
    frame_num 255, with MMCO 1 on frame_num 254 across the wrap and MMCO 3 on PicNum -1), still to 511 (no picture marks: changed
    stays 0), A again at 512, which predicts from the long-term picture 257 pictures later while picture 511, its short-term
    reference, has frame_num 255 too."""
    inv, yy = grey_table(), np.arange(h)[:, None] + np.zeros(w, np.int64)
    a, b = grey(w, h, inv, np.where(yy < h // 2, 60, 180)), grey(w, h, inv, np.where(yy < h // 2, 200, 40))
    return [a] * 256 + [b] * 256 + [a]


def ltr_cases():
    """The long-term reference (B2V_FLAG_LONG_TERM_REF, §5.13): the configurations of both files with the flag on.  Each reaches
    what LTR_TARGETS names for it."""
    w, h = 320, 192
    pan = [waves(128, 64, t, [(0, 64, 24, 1.25)], amp=30) for t in range(6)]
    return [("ltr_popup", S.Config(w, h, qp=26, flags=LTR), LC.popup(w, h)[0], (0,), None, 0),
            ("ltr_alt_tab_wide", S.Config(w, h, qp=26, flags=LTR | WIDE), LC.alt_tab(w, h)[0], (0,), None, 0),
            # two short popups, an IDR requested at 6 and a gop of 5 (an IDR at 11): no override after an IDR, the rule starting again
            ("ltr_cbr_idr_gop", S.Config(w, h, rc_mode=S.CBR, kbps=2000, fps=30.0, gop=5, flags=LTR),
             LC.popup(w, h, 2, 2, 2)[0] * 2, (0, 6), None, 0),
            # still, then bars of period 16 moving 8 px per picture (and of period 16.5 moving 8.25): picture 2 marks picture 1, and
            # picture 3 repeats picture 1, its vectors from picture 2 (the bars' half period either way)
            ("ltr_both_exits", S.Config(160, 96, qp=40, flags=LTR),
             [waves(160, 96, t, [(0, 48, 16, 8), (48, 96, 16.5, 8.25)], amp=20) for t in (0, 0, 1, 2, 3)], (0,), None, 0),
            ("ltr_pcm_noise_qp0_4", S.Config(64, 48, qp=0, flags=LTR), [synth.noise(64, 48, s) for s in (5, 5, 6, 7, 8)], (0,),
             [0, 0, 2, 4, 4], 0),
            ("ltr_frame_num_wrap", S.Config(48, 32, qp=26, flags=LTR), wrap_content(48, 32), (0,), None, 0),
            ("droppable_fractional_pan", S.Config(128, 64, qp=22, flags=LS.FLAG_DROPPABLE), pan, (0,), None, 0)]


def bars_over_texture(w, h, shifts, period=3, amp=40, seed=7):
    """BGRA pictures of vertical bars (a cosine of `period` px) over a weak non-periodic texture (random cosines of 5..40 px, about
    ±12 levels), both constant down each column.  Picture t holds the bars shifted left by shifts[t][0] px and the texture by
    shifts[t][1] px: where the two shifts of a step differ by a whole period, the bars alone match at a vector the texture does not."""
    rng = np.random.default_rng(seed)
    comps = [(rng.uniform(5, 40), rng.uniform(0, 2 * np.pi)) for _ in range(6)]
    x = np.arange(w, dtype=np.float64)
    out, inv = [], grey_table()
    for a, b in shifts:
        tex = sum(np.cos(2 * np.pi * (x + b) / p + ph) for p, ph in comps) * 4
        row = 128 + amp * np.cos(2 * np.pi * (x + a) / period) + tex
        out.append(grey(w, h, inv, np.repeat(np.rint(row).astype(np.int64)[None, :], h, 0)))
    return out


def smooth_texture_pan(w, h, n, v, seed=9):
    """n BGRA pictures of a smooth 2-D texture (random plane waves of 6..30 px) moving by v px per picture, fractional allowed (content
    at (x, y) was at (x, y) + v one picture earlier)."""
    rng = np.random.default_rng(seed)
    waves_ = [(rng.uniform(6, 30), rng.uniform(0, 2 * np.pi), rng.uniform(0, 2 * np.pi)) for _ in range(8)]
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    inv = grey_table()
    out = []
    for t in range(n):
        X, Y = xx + t * v[0], yy + t * v[1]
        luma = 128 + sum(12 * np.cos(2 * np.pi * (X * np.cos(th) + Y * np.sin(th)) / p + ph) for p, th, ph in waves_)
        out.append(grey(w, h, inv, np.clip(np.rint(luma), 16, 235).astype(np.int64)))
    return out


def noise_window_scroll(w, h, n, box, seed=21):
    """n BGRA desktop pictures scrolling up 3 px per picture with a window of fresh grey noise (new every picture) at box = (x, y,
    width, height): new content next to moving content."""
    rng = np.random.default_rng(seed)
    inv = grey_table()
    out = []
    for t in range(n):
        f = synth.desktop(w, h + 3 * n, 0)[3 * t:3 * t + h].copy()
        x, y, bw, bh = box
        f[y:y + bh, x:x + bw] = grey(bw, bh, inv, rng.integers(16, 236, (bh, bw)))
        out.append(f)
    return out


def motion_cases():
    """The motion search after the lean pass (§5.3): each reaches what assert_targets names for it."""
    # droppable: picture 2 (two back from picture 0) moves 2.75 px, so its vectors are 11 quarter samples; picture 3 (from picture 2)
    # moves the bars 2 px and the texture -1 px: the halved predictor 6 rounds to the candidate 2, where only the bars match — a strict
    # local minimum whose refinement codes a vector the search (at -1) never finds; halving toward zero (5) gives the candidate 1
    return [("droppable_scaled_alias", S.Config(128, 64, qp=30, flags=LS.FLAG_DROPPABLE),
             bars_over_texture(128, 64, [(0, 0), (0, 0), (2.75, 2.75), (4.75, 1.75)]), (0,), None, 0),
            # a fractional pan at QP 22: the previous vector is fractional, its full-sample candidate hits inside the picture, and the
            # refinement moves it (the lean pass must leave such a hit to the search pass)
            ("fractional_pan_qp22", S.Config(128, 64, qp=22), [waves(128, 64, t, [(0, 64, 24, 1.25)], amp=30) for t in range(5)],
             (0,), None, 0),
            # 13.25 px across and 5.5 px up per picture: searched vectors at the refinement gate's edge, |dx| = 13
            ("texture_pan_13", S.Config(160, 96, qp=26), smooth_texture_pan(160, 96, 3, (13.25, -5.5)), (0,), None, 0),
            # fresh noise next to a scroll: anchors inside the noise raise the new-content flag, their groups run the reduced search
            ("noise_window_scroll", S.Config(192, 128, qp=26), noise_window_scroll(192, 128, 3, (48, 32, 96, 64)), (0,), None, 0),
            # the coarse search's band edges with wide motion: each band's bottom group matches best one decimated row past its band,
            # 20 px across, so that a coarse search looking there moves the anchor's second window (and its coded vector)
            ("wide_band_bottoms", S.Config(128, 208, qp=26, stripe_rows=5, flags=WIDE), band_bottom_scroll(128, 208, 5, sx=20), (0,),
             None, 5)]


def directional(w, h, seed=1, tile=16):
    """BGRA picture of tile x tile squares, each an oriented pattern in two random colours: stripes of period 3..12 px, a step or a
    ramp, at one of eight orientations (multiples of 22.5°) through a point near the tile's centre."""
    rng = np.random.default_rng(seed)
    f = np.zeros((h, w, 4), np.uint8)
    f[..., 3] = 255
    for ty in range(0, h, tile):
        for tx in range(0, w, tile):
            yy, xx = np.mgrid[0:min(tile, h - ty), 0:min(tile, w - tx)].astype(np.float64)
            th = rng.integers(8) * np.pi / 8
            u = (xx - tile / 2 + rng.uniform(-2, 2)) * np.cos(th) + (yy - tile / 2 + rng.uniform(-2, 2)) * np.sin(th)
            kind = rng.integers(3)
            if kind == 0:
                v = 0.5 + 0.5 * np.cos(2 * np.pi * u / rng.uniform(3, 12))
            elif kind == 1:
                v = (u > 0).astype(np.float64)
            else:
                v = (u - u.min()) / max(np.ptp(u), 1)
            c0, c1 = rng.integers(0, 256, 3), rng.integers(0, 256, 3)
            f[ty:ty + tile, tx:tx + tile, :3] = np.rint(c0 + (c1 - c0) * v[..., None]).astype(np.uint8)
    return f


def flat(w, h):
    """BGRA picture of flat areas: mid grey on the left, a flat colour on the right, a dark grey band across the bottom."""
    f = np.full((h, w, 4), 255, np.uint8)
    f[:, :w // 2, :3] = 128
    f[:, w // 2:, :3] = (40, 160, 220)
    f[h - 16:, :, :3] = 60
    return f


def dots(w, h):
    """BGRA mid-grey picture with one 2x2 dot per macroblock, its amplitude rising by 1 from 1 in raster order: Intra16x16 SADs of
    4 per level step, either side of the Intra4x4 gate at small λ."""
    luma = np.full((h, w), 120, np.int64)
    for a in range((h // 16) * (w // 16)):
        y, x = 16 * (a // (w // 16)) + 5, 16 * (a % (w // 16)) + 9
        luma[y:y + 2, x:x + 2] += a + 1
    return grey(w, h, grey_table(), luma)


def noise_ramp(w, h, amp, seed=0, base=None):
    """BGRA grey picture: `base` (a luma plane; mid grey when None) plus uniform noise whose amplitude rises linearly from amp[0] at
    the left edge to amp[1] at the right edge."""
    rng = np.random.default_rng(seed)
    a = np.linspace(amp[0], amp[1], w)[None, :]
    luma = (np.full((h, w), 126, np.int64) if base is None else base) + np.rint(a * rng.uniform(-1, 1, (h, w))).astype(np.int64)
    return grey(w, h, grey_table(), np.clip(luma, 16, 235)), luma


def pcm_boundary_frames(w, h):
    """An IDR picture and a P picture whose macroblocks reach the I_PCM limit of §5.7 in a ramp across the picture (coded at QP 4
    and 0): noise of amplitude 50..110, then the same with fresh noise of amplitude 30..90 added."""
    f0, luma = noise_ramp(w, h, (50, 110), seed=1)
    f1, _ = noise_ramp(w, h, (30, 90), seed=2, base=np.clip(luma, 16, 235))
    return [f0, f1]


def intra_cases():
    """The intra decision (§5.2) and the I_PCM rule (§5.7) in both directions: each reaches what assert_targets names for it."""
    cut = SC.FLAG_SCENE_CUT
    d64 = directional(64, 48, 3)
    return [("intra_directional_qp26", S.Config(160, 96, qp=26), [directional(160, 96, 1)], (0,), None, 0),
            ("intra_directional_qp40", S.Config(160, 96, qp=40), [directional(160, 96, 1)], (0,), None, 0),
            ("intra_flat", S.Config(96, 64, qp=26), [flat(96, 64)], (0,), None, 0),
            ("intra_gate_dots", S.Config(128, 80, qp=10), [dots(128, 80)], (0,), None, 0),
            ("intra_slices3_crop", S.Config(136, 72, qp=30, idr_slice_mbs=3), [directional(136, 72, 2)] * 2, (0,), None, 0),
            ("intra_qp0", S.Config(64, 48, qp=0), [d64], (0,), None, 0),
            ("intra_qp10", S.Config(64, 48, qp=10), [d64], (0,), None, 0),
            ("intra_qp51", S.Config(64, 48, qp=51), [d64], (0,), None, 0),
            ("pcm_boundary", S.Config(320, 64, qp=0), pcm_boundary_frames(320, 64), (0,), [4, 0], 0),
            ("scut_switches_qp26", S.Config(160, 96, qp=26, flags=cut), SC.switches(160, 96), (0,), None, 0),
            ("scut_switches_ltr_qp36", S.Config(160, 96, qp=36, flags=cut | LTR), SC.switches(160, 96), (0,), None, 0),
            ("scut_noise_qp0_4", S.Config(64, 48, qp=0, flags=cut),
             [synth.desktop(64, 48)] * 2 + [synth.noise(64, 48, s) for s in (5, 6)], (0,), [0, 0, 2, 4], 0)]


def assert_targets(name, st):
    """What each case is there for, from the parsed streams and the model: a case that drifts away from its target fails."""
    ex = st.exits
    if name in ("pcm_noise_qp0_4", "wide_pcm_noise_qp0_4"):
        assert st.kinds.get("I_PCM", 0) > 0, st.kinds
    if name == "paintover_burst":
        assert st.kinds.get("P_L0_16x16", 0) > 0        # the burst re-codes the still at the paint-over QP
    if name in ("ltr_popup", "ltr_alt_tab_wide"):
        assert st.marks and ex.get("long-term", 0) > 0, (st.marks, ex)
    if name == "ltr_popup":
        assert st.skip_next_to_lt > 0, ex
    if name == "ltr_cbr_idr_gop":
        assert any(k > 6 for _, k in st.marks) and any(k < 6 for _, k in st.marks), st.marks
    if name == "ltr_both_exits":
        assert ex.get("predictor lean", 0) > 0 and ex.get("long-term over edge predictor", 0) > 0, ex
    if name == "ltr_pcm_noise_qp0_4":
        assert st.pcm_two_refs > 0, (st.kinds, st.marks)
    if name == "ltr_frame_num_wrap":
        assert st.mark_at_fn0 and st.mmco1_wrap and st.lt_age > 256 and st.lt_fn_twin > 0, \
            (st.marks, st.mark_at_fn0, st.mmco1_wrap, st.lt_age, st.lt_fn_twin)
    if name == "droppable_fractional_pan":
        assert st.scaled > 0, ex
    # the search half of §5.3: every path M.decide restates, and the rules whose mistakes only these cases expose
    want = {"qp26": ["refined search", "anchor predictor"], "pcm_noise_qp0_4": ["reduced search"],
            "wide_scroll250_tall": ["second window"], "wide_band_bottoms": ["second window"],
            "droppable_scaled_alias": ["scaled rounding decides", "refined predictor"],
            "fractional_pan_qp22": ["refined predictor", "refinement moves an inside fractional hit"],
            "texture_pan_13": ["refined at |d| = 13", "anchor candidate rounded up"],
            "noise_window_scroll": ["reduced search at |dy| = 2", "refined with SAD >= 4096"]}
    for path in want.get(name, []):
        assert st.paths.get(path, 0) > 0, (path, st.paths)
    # the intra decision: every mode and branch of §5.2 where a mistake in it changes what is coded
    intra = (st.i4_row0, st.i4_rows, st.i16_modes, st.chroma_modes, st.i4_untried, st.compared, st.ties, st.slice_starts)
    if name.startswith("intra_directional"):
        assert st.i4_rows == set(range(9)) and st.i4_row0 == {1, 2, 8}, intra
        assert st.i16_modes == {1, 2} and st.chroma_modes == {0, 1}, intra
        assert st.compared.get("I_NxN", 0) > 0 and st.compared.get("I_16x16", 0) > 0, intra
    if name == "intra_flat":
        assert st.i4_untried > 0 and st.ties.get("I16 H over DC", 0) > 0 and st.ties.get("chroma DC over H", 0) > 0, intra
    if name == "intra_gate_dots":                    # the gate shuts Intra4x4 out where it would have won
        assert st.gate_decides > 0 and st.compared.get("I_NxN", 0) > 0, intra
    if name == "intra_slices3_crop":
        assert st.slice_starts >= 10, intra          # 9 macroblocks a row in slices of 3: two slice starts inside each of 5 rows
    if name in ("intra_qp0", "intra_qp10"):          # rd_lambda 1, λ 1: both kinds kept after a comparison
        assert st.compared.get("I_NxN", 0) > 0 and st.compared.get("I_16x16", 0) > 0, intra
    if name == "intra_qp51":                           # rd_lambda 6963, λ 57: the comparison made, Intra16x16 kept
        assert st.compared.get("I_16x16", 0) > 0, intra
    if name == "pcm_boundary":     # coded and I_PCM macroblocks within 100 bits of the limit, on either side of it, intra and inter
        for t in "IP":
            assert 3100 <= st.max_coded[t] and st.min_pcm[t] is not None and st.min_pcm[t] <= 3300, (t, st.max_coded, st.min_pcm, st.kinds)
    if name.startswith("scut_"):
        assert st.cut_pictures > 0, st.kinds
    if name == "scut_noise_qp0_4":
        assert st.cut_pcm > 0, st.kinds


CASES = cases()


def run_case(encode, case):
    _, cfg, frames, idr_at, qps, stripe_rows = case
    e = encode(cfg, frames, idr_at, qps)
    st = check_encoded(e, stripe_rows)
    return e, st


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_decisions(case):
    e, st = run_case(encode_oracle, case)
    check_recon(e, st)
    assert st.pictures >= len(case[2])
    assert_targets(case[0], st)


def nal_ref_idc(au):
    """nal_ref_idc of the first slice of an access unit."""
    return next(n[0] >> 5 & 3 for n in split_annexb(au) if n[0] & 31 in (1, 5))


# The decisions' wide-motion cases (the long-term reference's left out: its coarse search is the wide oracle's), and three more for the coarse search alone: mbw % 4 = 2 in bands of 5 rows at QP 51 (the
# largest λ: most groups stay below the early exit), mbw % 4 = 3 at QP 0 (λ = 1: nearly every group searches), 2x2-blocky
# noise moved 124 px left and 256 px down, whose only match is the coarse window's corner (dx = 31, dy = -64), and noise
# scrolled in bands of 5 rows whose bottom groups match best one decimated row past the band.
COARSE_CASES = [c for c in CASES if c[1].flags & WIDE and not c[1].flags & LTR] + [
    ("coarse_drag_stripes5_qp51", S.Config(160, 144, qp=51, stripe_rows=5, flags=WIDE),
     [WC.drag(160, 144, t, (-30, 22), (90, 10), 64, 64) for t in range(4)], (0,), None, 5),
    ("coarse_scroll_qp0", S.Config(240, 208, qp=0, flags=WIDE), [WC.desktop_scroll(240, 208, t, 60) for t in range(3)], (0,), None, 0),
    ("coarse_noise_corner", S.Config(192, 448, qp=26, flags=WIDE), [blocky_noise(192, 448, 0, 256), blocky_noise(192, 448, 124, 0)],
     (0,), None, 0),
    ("coarse_band_bottoms", S.Config(128, 208, qp=26, stripe_rows=5, flags=WIDE), band_bottom_scroll(128, 208, 5), (0,), None, 5)]


@pytest.mark.parametrize("case", COARSE_CASES, ids=[c[0] for c in COARSE_CASES])
def test_oracle_coarse_search(case):
    """The decimated plane of every picture equals the model's decimation of its source, and at every macroblock the coarse table
    equals the model's coarse search (None included: non-anchors, still groups, IDR pictures) between the decimated sources of the
    picture and of its reference (the last reference picture: two back after a droppable one)."""
    _, cfg, frames, idr_at, qps, stripe_rows = case
    seen = []
    e = encode_oracle(cfg, frames, idr_at, qps,
                      each=lambda i, enc, bands: seen.append((enc.decimated(), enc.coarse(), enc.recon()[0].copy(),
                                                              nal_ref_idc(bands[0][1]) if bands else 1)))
    mbw, mbh = e.cw // 16, e.ch // 16
    rows = stripe_rows or mbh
    ref, searched = None, 0
    for i, (dec, coarse, recon, ref_idc) in enumerate(seen):
        y = e.sources[i][0]
        assert np.array_equal(dec, M.decimate(y)), f"picture {i}: decimated plane"
        if i in idr_at:
            assert all(v is None for row in coarse for v in row), f"picture {i}: an IDR picture with coarse vectors"
        else:
            dref, yref = M.decimate(e.sources[ref][0]), seen[ref][2].astype(np.int64)
            dcur = M.decimate(y)
            for mby in range(mbh):
                r0 = mby // rows * rows
                for mbx in range(mbw):
                    x0, y0 = 16 * mbx, 16 * mby
                    sad0 = M.sad(y[y0:y0 + 16, x0:x0 + 16], yref[y0:y0 + 16, x0:x0 + 16])
                    want = M.coarse_search(dcur, dref, mbx, mby, mbw, r0, min(r0 + rows, mbh), sad0, cfg.qp if qps is None else qps[i])
                    assert coarse[mby][mbx] == want, f"picture {i} mb ({mbx},{mby}): coarse vector {coarse[mby][mbx]}, model {want}"
                    searched += want is not None
        if ref_idc:
            ref = i
    assert searched > 0


def test_oracle_decisions_720p_idr():
    """One 1280x720 IDR: the parser's cost at the largest size in the suite."""
    w, h = 1280, 720
    t0 = time.perf_counter()
    e, st = run_case(encode_oracle, ("720p", S.Config(w, h, qp=33), [synth.desktop(w, h, 0)], (0,), None, 0))
    assert st.kinds.get("I_NxN", 0) + st.kinds.get("I_16x16", 0) == 3600
    print(f"720p IDR: parse + model + checks {time.perf_counter() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ motion (§5.3)
class OracleEnc:
    """One CQP oracle encoder, picture by picture: encode() returns {band y_start: access unit} of the coded bands."""

    def __init__(self, w, h, qp, slice_rows=0, stripe_rows=0, wide=False):
        self.e = (WS.WideRefEncoder if wide else oracle.RefEncoder)(w, h, slice_rows)
        if stripe_rows:
            self.e.set_stripes(stripe_rows)
        if wide:
            self.e.set_wide_motion(True)
        self.qp, self.stripe_rows = qp, stripe_rows

    def encode(self, frame, idr):
        au = self.e.encode_bgra(frame, idr, qp=self.qp)
        if not self.stripe_rows:
            return {0: au}
        return {k * self.stripe_rows * 16: au[o:o + n] for k, (o, n, coded) in enumerate(self.e.stripe_table()) if coded}

    def recon(self):
        return self.e.recon()

    def close(self):
        self.e.close()


def shifted(y, mv):
    """Luma plane y moved by the quarter-sample vector mv with the model's interpolation: sample (x, y) of the result is the
    prediction a decoder makes from y for vector mv at (x, y)."""
    h, w = y.shape
    out = np.zeros((h, w), np.int64)
    for y0 in range(0, h, 16):
        for x0 in range(0, w, 16):
            out[y0:y0 + 16, x0:x0 + 16] = M.luma_inter(y, x0, y0, mv)
    return out


# Full-sample extremes of the window, interior full-sample shifts, and half- and quarter-sample shifts with |d| <= 13.
RECOVERY_SHIFTS = [(-64, 0), (60, 0), (0, -64), (0, 64), (-64, 64), (20, -12), (10, -6), (-26, 18), (5, -3), (-51, 45), (47, -1)]
# Wide-range motion (quarter samples) on a wide, short picture: 16 and -17 px, just past the co-located window (16 px needs the
# second search: the co-located one ends at 15); the coarse window's edges -128 and +124 px across; (37, -53) px, not a multiple
# of 4; (-90.5, 20.25) px, fractional, its refinement gate open.  On a tall, narrow one: 252 px down, the coarse window's last row,
# and 255 px up, the end of the vector range.
WIDE_SHIFTS_ACROSS = [(64, 0), (-68, 0), (-512, 0), (496, 0), (148, -212), (-362, 81)]
WIDE_SHIFTS_DOWN = [(0, 1008), (0, -1020)]


def _interior(mbx, mby, mv, w, h, wide):
    """The macroblocks a search must resolve to exactly the shift mv.  The 48x48 window of §5.3 spans x0-16 .. x0+31 and y0-16 ..
    y0+31 around its centre; where it lies inside the picture nothing is clamped, and the refinement runs only for |d| <= 13,
    whose 6-tap support (-15 .. +31) stays inside the window.  Without wide motion the window is centred on the macroblock; with
    it, on the shift's full-sample vector (its x rounded down to a multiple of 4, as §5.3 stages a far candidate's window), and the
    macroblock's group, moved by the shift / 4 either way rounded, stays inside the decimated plane: the coarse search sees it."""
    fx, fy = ((mv[0] + 2) >> 2, (mv[1] + 2) >> 2) if wide else (0, 0)
    cx = fx & ~3
    if not (16 <= 16 * mbx + cx and 16 * mbx + cx + 32 <= w and 16 <= 16 * mby + fy and 16 * mby + fy + 32 <= h):
        return False
    if not wide:
        return True
    gx0, gy0 = 4 * (mbx // 4), 4 * (mby // 4)
    gx1, gy1 = min(gx0 + 4, w // 16), min(gy0 + 4, h // 16)
    return (16 * gx0 + 4 * (fx // 4) >= 0 and 16 * gx1 + 4 * -(-fx // 4) <= w and 16 * gy0 + 4 * (fy // 4) >= 0
            and 16 * gy1 + 4 * -(-fy // 4) <= h)


def motion_recovery(make_enc, qp=26, w=256, h=160, wide=False, shifts=RECOVERY_SHIFTS, gate_at=(3, 2)):
    """An IDR of 2x2-blocky mid-range luma noise, then for each shift a P picture built from the encoder's own reconstruction
    moved by the shift: every macroblock must come out with cbp 0, and every macroblock _interior() names must carry exactly the
    shift.  wide: with wide-range motion, where cbp 0 is asserted on those macroblocks only (a group whose block the shift moves
    out of the decimated plane has no coarse match, and its macroblocks may code a residual); and for a fractional shift on the
    anchors only: the others reach a far vector only through their anchor's, whose test accepts a full-sample SAD of at most
    4·96·λ, and an open refinement gate puts it above that.  A fractional shift's refinement gate is checked open at macroblock
    gate_at."""
    rng = np.random.default_rng(11)
    luma = rng.integers(96, 160, (h // 2, w // 2)).repeat(2, 0).repeat(2, 1)
    inv = grey_table()
    f0 = grey(w, h, inv, luma)
    enc = make_enc(w, h, qp, wide=wide)
    try:
        aus0 = enc.encode(f0, True)
        parser = StreamParser()
        parser.picture(aus0[0])
        ry, ruv = enc.recon()
        assert (ruv == 128).all()
        lam = M.LAMBDA[qp]
        mbw, mbh = w // 16, h // 16
        for mv in shifts:
            y1 = shifted(ry, mv)
            assert 16 <= y1.min() and y1.max() <= 235                   # no sample of the target is clipped by the CSC
            # the refinement gate of §5.3 is open for a fractional shift: full-sample SAD above 96·λ and below 8192
            if (mv[0] | mv[1]) & 3:
                fs, (x0, y0) = ((mv[0] + 2) >> 2, (mv[1] + 2) >> 2), (16 * gate_at[0], 16 * gate_at[1])
                assert _interior(*gate_at, mv, w, h, wide)
                s = M.sad(y1[y0:y0 + 16, x0:x0 + 16], M.luma_inter(ry, x0, y0, (4 * fs[0], 4 * fs[1])))
                assert M.EARLY_SAD_PER_LAMBDA * lam < s < M.REFINE_MAX_SAD, (mv, s)
            f1 = grey(w, h, inv, y1)
            enc.encode(f0, True)                                        # the same parameter sets: parsed once
            p = parser.picture(enc.encode(f1, False)[0])
            interior = 0
            for m in p.mbs:
                mbx, mby = m.addr % mbw, m.addr // mbw
                inside = _interior(mbx, mby, mv, w, h, wide)
                if wide and (mv[0] | mv[1]) & 3 and M.anchor_of(mbx, mby, mbw, 0, mbh) != (mbx, mby):
                    inside = False          # a far fractional vector is the anchors' alone: see the docstring
                if inside or not wide:
                    assert m.kind in ("P_Skip", "P_L0_16x16") and m.cbp == 0, (mv, mbx, mby, m.kind, m.cbp, m.mv)
                if inside:
                    assert m.mv == mv, (mv, mbx, mby, m.mv)
                    interior += 1
            assert interior == (mbw - 2) * (mbh - 2) if not wide else interior >= 4, (mv, interior)
    finally:
        enc.close()


def test_oracle_motion_recovery():
    motion_recovery(OracleEnc)


@pytest.mark.parametrize("w,h,shifts,gate_at", [(448, 128, WIDE_SHIFTS_ACROSS, (13, 1)), (96, 640, WIDE_SHIFTS_DOWN, None)],
                         ids=["across", "down"])
def test_oracle_wide_motion_recovery(w, h, shifts, gate_at):
    motion_recovery(OracleEnc, w=w, h=h, wide=True, shifts=shifts, gate_at=gate_at)


def search_optimality(make_enc, w, h, stripe_rows=0, qp=28, wide=False, shift=(-5, 7), blocky=False):
    """A cut to new structured content (a gradient with noise, or 2x2-blocky noise, still for one picture, then translated by
    `shift` px plus mild noise).  On the translated picture the anchors search (§5.3).  For every anchor the model shows did
    search — SAD(0,0) above 96·λ and the temporal predictor (its previous vector) more than 4·96·λ off — the documented cost of
    the coded vector is at most the brute-force minimum over the window, and equal to it when the vector is full-sample; and the
    coded vector is exactly the model's: the search's winner (M.search), refined (M.refine).
    wide: with wide-range motion, over the co-located window and the window around the model's coarse vector × 4 (when §5.3
    searches it), vectors outside the range left out, the winner of the two by cost, the co-located window on equal cost."""
    rng = np.random.default_rng(5)
    sx, sy = shift
    ox, oy = max(24, -sx), max(20, -sy)                                  # the still picture's corner in the content
    yy, xx = np.mgrid[0:oy + max(sy, 44) + h, 0:ox + max(sx, 40) + w]
    if blocky:
        base = rng.integers(40, 200, ((yy.shape[0] + 1) // 2, (xx.shape[1] + 1) // 2)).repeat(2, 0).repeat(2, 1)[:yy.shape[0], :xx.shape[1]]
    else:
        base = 40 + (xx * 3 + yy * 2) % 150 + rng.integers(0, 30, xx.shape)
    mild = lambda: rng.integers(-2, 3, (h, w))
    inv = grey_table()
    still = grey(w, h, inv, np.clip(base[oy:oy + h, ox:ox + w], 16, 235))
    moved = grey(w, h, inv, np.clip(base[oy + sy:oy + sy + h, ox + sx:ox + sx + w] + mild(), 16, 235))
    enc = make_enc(w, h, qp, stripe_rows=stripe_rows, wide=wide)
    try:
        streams = {}
        for i, f in enumerate([still, still, moved]):
            for y0, au in enc.encode(f, i == 0).items():
                streams.setdefault(y0, []).append(au)
    finally:
        enc.close()
    lam, checked, anchors, far = M.LAMBDA[qp], 0, 0, 0
    cw, ch = (w + 15) // 16 * 16, (h + 15) // 16 * 16
    sources = [source_nv12(f, cw, ch) for f in (still, still, moved)]
    for y0, aus in streams.items():
        pics = HSR.parse_stream(aus)             # a band whose still picture was all skipped is not sent: 2 pictures
        mbw, mbh = pics[-1].sps.mbw, pics[-1].sps.mbh
        band = [[p[y0 // k:(y0 + 16 * mbh) // k] for p, k in zip(s, (1, 2, 2))] for s in sources]
        st, recs = Stats(), []
        for i in range(len(pics) - 1):
            recs.append(check_picture(pics[i], recs, band[i], f"band {y0} picture {i}", st))
        rec = recs[-1]
        prev_mbs = pics[1].mbs if len(pics) == 3 else [Mb(a, 0, "P_Skip", qp) for a in range(mbw * mbh)]
        # the coded-size reference of the band (or picture): a band's stream clamps at the band's own edges
        ref = rec[0]
        cur = band[2][0].astype(np.int64)
        dec_cur, dec_ref = M.decimate(band[2][0]), M.decimate(band[1][0])      # the reference is picture 1, still
        early = M.EARLY_SAD_PER_LAMBDA * lam
        for m in pics[-1].mbs:
            mbx, mby = m.addr % mbw, m.addr // mbw
            if M.anchor_of(mbx, mby, mbw, 0, mbh) != (mbx, mby) or m.kind == "I_PCM":
                continue
            anchors += 1
            blk = cur[16 * mby:16 * mby + 16, 16 * mbx:16 * mbx + 16]
            costs = M.full_search(blk, ref, 16 * mbx, 16 * mby, qp)
            prev = prev_mbs[m.addr]
            pv = ((prev.mv[0] + 2) >> 2, (prev.mv[1] + 2) >> 2) if not prev.intra else None
            if costs[(0, 0)][0] <= early or (pv in costs and costs[pv][0] <= 4 * early):
                continue
            checked += 1
            v, s_, c_ = M.search(blk, ref, 16 * mbx, 16 * mby, qp)
            centre = (0, 0)
            if wide:
                coarse = M.coarse_search(dec_cur, dec_ref, mbx, mby, mbw, 0, mbh, costs[(0, 0)][0], qp)
                far_centre = M.second_window(coarse)
                if far_centre is not None:
                    costs.update(M.full_search(blk, ref, 16 * mbx, 16 * mby, qp, centre=far_centre))
                    v2, s2, c2 = M.search(blk, ref, 16 * mbx, 16 * mby, qp, centre=far_centre)
                    if c2 < c_:
                        v, s_, centre = v2, s2, far_centre
                    far += 1
            best = min(c for _, c in costs.values())
            pred = M.luma_inter(ref, 16 * mbx, 16 * mby, m.mv)
            cost = M.motion_cost(M.sad(blk, pred), m.mv, qp)
            if (m.mv[0] | m.mv[1]) & 3:
                assert cost <= best, (y0, mbx, mby, m.mv, cost, best)
            else:
                assert cost == best, (y0, mbx, mby, m.mv, cost, best)
            # exactly the search's winner, refined in its window
            want, _ = M.refine(blk, ref, 16 * mbx, 16 * mby, v, centre, s_, qp)
            assert m.mv == want, (y0, mbx, mby, m.mv, want, v, centre)
    assert anchors and checked >= 0.75 * anchors, (checked, anchors)
    assert far or not wide


@pytest.mark.parametrize("w,h,stripe_rows", [(130, 70, 0), (200, 112, 3)])
def test_oracle_search_optimality(w, h, stripe_rows):
    search_optimality(OracleEnc, w, h, stripe_rows)


# The cut translated by large vectors (px); in bands of 3 rows, whose edges clamp the coarse search; and 2x2-blocky noise moved 256 px
# down, one row past the vector range: the coarse window's first row (dy = -64) is its only decimated match.
WIDE_OPTIMALITY = [(192, 176, 0, (-45, 70), False), (256, 96, 0, (90, -30), False), (256, 144, 3, (-70, 21), False),
                   (64, 448, 0, (0, -256), True)]


@pytest.mark.parametrize("w,h,stripe_rows,shift,blocky", WIDE_OPTIMALITY)
def test_oracle_wide_search_optimality(w, h, stripe_rows, shift, blocky):
    search_optimality(OracleEnc, w, h, stripe_rows, wide=True, shift=shift, blocky=blocky)


# ------------------------------------------------------------------------------------------------ level_idc (Table A-1)
@pytest.mark.parametrize("w,h,stripe_rows", [(3840, 64, 0), (3840, 2160, 8)])
def test_wide_pictures_and_bands_carry_a_level_that_holds_them(w, h, stripe_rows):
    """A 3840x64 picture (240 macroblocks per row) and each 240x8 band of a striped 4K picture exceed the sqrt(8 * MaxFS) = 169
    width bound of level 3.1 although they fit its MaxFS; their SPS must name a level that holds them."""
    enc = oracle.RefEncoder(w, h, 0)
    if stripe_rows:
        enc.set_stripes(stripe_rows)
    f = np.zeros((h, w, 4), np.uint8)
    au = enc.encode_bgra(f, True, qp=40)
    from tests.h264_syntax import parse_sps, split_annexb, unescape
    spss = [parse_sps(unescape(n)) for n in split_annexb(au) if n[0] & 31 == 7]
    assert len(spss) == (-(-h // (16 * stripe_rows)) if stripe_rows else 1)
    for sps in spss:
        assert level_ok(sps.level_idc, sps.mbw, sps.mbh), (sps.level_idc, sps.mbw, sps.mbh)
        assert sps.level_idc == smallest_level(sps.mbw, sps.mbh)


@pytest.mark.parametrize("w,h,level", [(16, 16, 31), (7680, 16, 51), (16, 4320, 51), (7680, 4320, 62), (2704, 16, 31),
                                       (2720, 16, 42), (4208, 16, 42), (4224, 16, 51), (3840, 1472, 51), (3840, 1488, 52),
                                       (3840, 2160, 52), (4096, 2304, 52), (4112, 2304, 62), (1920, 1080, 42), (1280, 720, 31)])
def test_level_rule_over_accepted_extremes(w, h, level):
    """The rule, walked through the sizes the library accepts (even, 16..7680 x 16..4320) and the edges of each rung: every
    size fits the ladder, at its first rung whose cap and Table A-1 bounds hold it — checked in the SPS the oracle writes.
    7680x16 (480 macroblocks per row) exceeds 4.2's width bound of 263 and fits 5.1's of 543; 3840x1472 (22080 macroblocks)
    is 5.1 and 3840x1488 (22320) is past 5.1's cap; 4112x2304 (37008) is past MaxFS of 5.2."""
    assert smallest_level(-(-w // 16), -(-h // 16)) == level
    enc = oracle.RefEncoder(w, h, 0)
    from tests.h264_syntax import parse_sps, split_annexb, unescape
    f = np.zeros((h, w, 4), np.uint8)
    au = enc.encode_bgra(f, True, qp=51)
    sps = parse_sps(unescape(split_annexb(au)[0]))
    assert sps.level_idc == level and (sps.width, sps.height) == (w, h)
