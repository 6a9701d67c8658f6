"""tests/h264_syntax.py's independent reader, extended to the reference-picture syntax of the long-term reference
(B2V_FLAG_LONG_TERM_REF): num_ref_idx_active_override, ref_idx_l0, adaptive dec_ref_pic_marking (7.3.3, 7.3.3.3, 7.3.5.1), motion-
vector prediction and P_Skip with refIdx (8.4.1.1, 8.4.1.3), and a decoded picture buffer (8.2.4, 8.2.5: sliding window and
memory_management_control_operation 1 to 6) that follows the reference marking.  Written from the Recommendation like the reader it
extends, whose SPS / PPS parsers, bit reader, residual coding and neighbour rules it reuses unchanged; it shares no code with oracle/
or selkies_b200/.

`parse_stream(aus)` returns what h264_syntax.parse_stream does, and besides: every P picture carries its RefPicList0
(`Picture.ref_list`: decoding-order indices) and the long-term frames after its marking (`Picture.long_term`), every inter
macroblock its `ref_idx` and the picture it predicts from (`Mb.ref_pic`), every coded macroblock the bits of its header
(`Mb.header_bits`: everything before the residual), and a slice header its override (`num_ref_idx_active`)
and its marking operations (`mmco`: (op, args...) tuples) when it has them.  The DPB raises when a stream marks more reference
frames than max_num_ref_frames or names a picture it does not hold."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

from tests import h264_syntax as HS
from tests.h264_syntax import SyntaxError_


@dataclass
class Mb(HS.Mb):
    ref_idx: int = 0             # ref_idx_l0 of an inter macroblock (0 for P_Skip)
    ref_pic: int = -1            # inter macroblock: decoding-order index of the picture RefPicList0[ref_idx] names
    header_bits: int = 0         # macroblock_layer() bits before the residual: mb_type .. mb_qp_delta (0 for P_Skip and I_PCM)


@dataclass
class Picture(HS.Picture):
    index: int = 0               # decoding order in the stream
    ref_list: list = field(default_factory=list)     # P pictures: RefPicList0 as decoding-order indices (8.2.4.2.1)
    long_term: list = field(default_factory=list)    # after this picture's marking: indices of the long-term reference frames


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
            out.append((True, m.ref_idx, m.mv))
    return out


def mv_pred(state, cur, ref_idx):
    """8.4.1.3: the luma motion vector predictor of a 16x16 partition with refIdxL0 = ref_idx; a neighbour with another refIdx keeps
    its vector in the median but is not a match."""
    (avA, rA, mA), (avB, rB, mB), (avC, rC, mC) = _mv_neighbours(state, cur)
    if not avB and not avC and avA:
        rB, mB, rC, mC = rA, mA, rA, mA
    refs = [rA == ref_idx, rB == ref_idx, rC == ref_idx]
    if sum(refs) == 1:
        return (mA, mB, mC)[refs.index(True)]
    return tuple(int(np.median([mA[i], mB[i], mC[i]])) for i in range(2))


def mv_skip(state, cur):
    """8.4.1.1: the P_Skip motion vector (refIdx 0)."""
    a, b_ = state.nb(cur, -1, 0), state.nb(cur, 0, -1)
    if a is None or b_ is None:
        return (0, 0)
    for m in (a, b_):
        if not m.intra and m.ref_idx == 0 and m.mv == (0, 0):
            return (0, 0)
    return mv_pred(state, cur, 0)


def _macroblock_layer(b, state, m: Mb, slice_p: bool, qp: int):
    """h264_syntax._macroblock_layer with ref_idx_l0 and refIdx-aware prediction"""
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
            pm = HS._i4_pred_mode(state, m, blk)
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
        if state.num_ref > 1:                            # ref_idx_l0: te(v), range num_ref_idx_l0_active - 1 (9.1)
            m.ref_idx = 1 - b.u(1) if state.num_ref == 2 else b.ue()
            if m.ref_idx >= state.num_ref:
                raise SyntaxError_("ref_idx_l0 out of range")
        m.mvd = (b.se(), b.se())
        p = mv_pred(state, m, m.ref_idx)
        m.mv = (p[0] + m.mvd[0], p[1] + m.mvd[1])
        m.skip_mv = mv_skip(state, m)
    if m.kind != "I_16x16":
        m.cbp = (HS.CBP_INTRA if m.intra else HS.CBP_INTER)[b.ue()]
    if m.cbp or m.kind == "I_16x16":
        qp = (qp + b.se() + 52) % 52                     # 7.4.5 mb_qp_delta
    m.qp = qp
    m.header_bits = b.pos - start
    HS._residual(b, state, m, m.kind == "I_16x16")
    m.bits = b.pos - start
    return qp


def _dec_ref_pic_marking(b):
    """7.3.3.3 with adaptive_ref_pic_marking_mode_flag = 1: the operations up to MMCO 0"""
    ops = []
    while True:
        op = b.ue()
        if op == 0:
            return ops
        if op > 6:
            raise SyntaxError_(f"memory_management_control_operation {op}")
        args = []
        if op in (1, 3):
            args.append(b.ue())                          # difference_of_pic_nums_minus1
        if op == 2:
            args.append(b.ue())                          # long_term_pic_num
        if op in (3, 6):
            args.append(b.ue())                          # long_term_frame_idx
        if op == 4:
            args.append(b.ue())                          # max_long_term_frame_idx_plus1
        ops.append((op, *args))


def parse_slice(rbsp: bytes, nal_type: int, nal_ref_idc: int, sps, pps: dict, state, slice_idx: int):
    """h264_syntax.parse_slice with the override (up to two references) and adaptive marking"""
    b = HS.Bits(rbsp)
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
    state.num_ref = pps["num_ref_idx_l0"]
    if slice_type == 0:
        if b.u(1):                                       # num_ref_idx_active_override_flag
            hdr["num_ref_idx_active"] = state.num_ref = b.ue() + 1
            if state.num_ref > 2:
                raise SyntaxError_("more than two reference indices")
        if b.u(1):
            raise SyntaxError_("ref_pic_list_modification is outside the subset")
    if nal_ref_idc:
        if idr:
            hdr["no_output_of_prior_pics"], hdr["long_term_reference_flag"] = b.u(1), b.u(1)
        elif b.u(1):                                     # adaptive_ref_pic_marking_mode_flag
            hdr["mmco"] = _dec_ref_pic_marking(b)
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
    """Parses the access units of one stream in decoding order, with its decoded picture buffer."""

    def __init__(self):
        self.sps = self.pps = None
        self.nal_types = []
        self.count = 0
        self.short = []                  # short-term reference frames: (frame_num, decoding index)
        self.long = {}                   # long-term reference frames: LongTermFrameIdx -> decoding index
        self.max_lt_idx = -1             # MaxLongTermFrameIdx ("no long-term frame indices": -1)

    def _pic_num(self, fn, cur_fn):
        """8.2.4.1: PicNum of a short-term frame (FrameNumWrap)"""
        return fn - (1 << self.sps.log2_max_frame_num) if fn > cur_fn else fn

    def _ref_list(self, pic, num_ref):
        """8.2.4.2.1: short-term frames by descending PicNum, then long-term frames by ascending LongTermPicNum"""
        st = sorted(self.short, key=lambda e: -self._pic_num(e[0], pic.frame_num))
        return ([i for _, i in st] + [self.long[k] for k in sorted(self.long)])[:num_ref]

    def _mark(self, pic, hdr, ref_idc):
        """8.2.5: the reference marking after a reference picture is decoded"""
        if not ref_idc:
            return
        if pic.idr:
            if hdr.get("long_term_reference_flag"):
                self.short, self.long, self.max_lt_idx = [], {0: pic.index}, 0
            else:
                self.short, self.long, self.max_lt_idx = [(pic.frame_num, pic.index)], {}, -1
            return
        current_long = False
        if "mmco" in hdr:
            for op, *a in hdr["mmco"]:
                if op in (1, 3):
                    x = pic.frame_num - (a[0] + 1)
                    hit = [e for e in self.short if self._pic_num(e[0], pic.frame_num) == x]
                    if not hit:
                        raise SyntaxError_(f"MMCO {op}: no short-term frame with PicNum {x}")
                    self.short.remove(hit[0])
                    if op == 3:
                        if a[1] > self.max_lt_idx:
                            raise SyntaxError_("MMCO 3: long_term_frame_idx above MaxLongTermFrameIdx")
                        self.long[a[1]] = hit[0][1]
                elif op == 2:
                    if a[0] not in self.long:
                        raise SyntaxError_(f"MMCO 2: no long-term frame {a[0]}")
                    del self.long[a[0]]
                elif op == 4:
                    self.max_lt_idx = a[0] - 1
                    self.long = {k: v for k, v in self.long.items() if k <= self.max_lt_idx}
                elif op == 5:
                    self.short, self.long, self.max_lt_idx = [], {}, -1
                elif op == 6:
                    self.long[a[0]] = pic.index
                    current_long = True
        elif len(self.short) + len(self.long) >= max(self.sps.max_num_ref_frames, 1):
            if not self.short:
                raise SyntaxError_("sliding window with no short-term frame")
            self.short.remove(min(self.short, key=lambda e: self._pic_num(e[0], pic.frame_num)))
        if not current_long:
            self.short.append((pic.frame_num, pic.index))
        if len(self.short) + len(self.long) > max(self.sps.max_num_ref_frames, 1):
            raise SyntaxError_("more reference frames than max_num_ref_frames")

    def picture(self, au: bytes) -> Picture:
        pic, state, ref_idc = None, None, 0
        for nal in HS.split_annexb(au):
            if nal[0] & 0x80:
                raise SyntaxError_("forbidden_zero_bit")
            ref_idc, t = nal[0] >> 5 & 3, nal[0] & 31
            self.nal_types.append(t)
            rbsp = HS.unescape(nal)
            if t == 7:
                self.sps = HS.parse_sps(rbsp)
            elif t == 8:
                self.pps = HS.parse_pps(rbsp)
            elif t in (1, 5):
                if state is None:
                    state = HS._PicState(self.sps)
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
        if any(("mmco" in h) != ("mmco" in pic.headers[0]) or h.get("mmco") != pic.headers[0].get("mmco") for h in pic.headers):
            raise SyntaxError_("the slices of a picture disagree on its marking")
        pic.mbs = state.mbs
        pic.index = self.count
        self.count += 1
        if not pic.idr:
            pic.ref_list = self._ref_list(pic, pic.headers[0].get("num_ref_idx_active", self.pps["num_ref_idx_l0"]))
            for m in pic.mbs:
                if not m.intra:
                    if m.ref_idx >= len(pic.ref_list):
                        raise SyntaxError_("ref_idx_l0 names no reference picture")
                    m.ref_pic = pic.ref_list[m.ref_idx]
        self._mark(pic, pic.headers[0], ref_idc)
        pic.long_term = [self.long[k] for k in sorted(self.long)]
        return pic


def parse_stream(aus):
    p = StreamParser()
    return [p.picture(bytes(a)) for a in aus]
