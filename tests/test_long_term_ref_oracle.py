"""The long-term reference picture (B2V_FLAG_LONG_TERM_REF) in the oracle.  Every stream decodes with libavcodec to the oracle's
reconstructions, over CQP and CBR, wide motion on and off, paint-over, IDR requests and a gop, a resize, an odd cropped size and
scaling.  The independent syntax model (tests/h264_syntax_refs.py, on tests/h264_syntax.py) finds the SPS values, the marking operations in exactly the pictures
the rule of tests/h264_model.py names (on its own changed(k)), the override exactly while a long-term picture exists, and refIdx-1 macroblocks only with the zero vector, never as
P_Skip, within the zero-motion threshold of the long-term picture its DPB names.  max_num_ref_frames 2 fits MaxDpbFrames at every
level the encoder writes.  The flag cuts the bytes of the pictures on which content comes back and costs the existing contents at
most 2 %."""
import numpy as np
import pytest

import oracle
from oracle import avdec
from oracle.ltr import LongTermRefEncoder
from tests import h264_model as M
from tests import h264_syntax as HS
from tests import h264_syntax_refs as HSR
from tests import ltr_content as LC
from tests import synth


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def _encode(frames, ltr=True, wide=False, w=None, h=None, idr_at=(), paint=None, **kw):
    h_, w_ = frames[0].shape[:2]
    w, h = w or w_, h or h_
    e = LongTermRefEncoder(w, h)
    if paint:
        e.set_paintover(*paint)
    e.set_wide_motion(wide)
    e.set_long_term_ref(ltr)
    aus, recs, states, lts = [], [], [], []
    for i, f in enumerate(frames):
        lts.append(e.long_term_picture() if ltr else None)      # what picture i may predict from
        aus.append(e.encode_bgra(f, i == 0 or i in idr_at, **kw))
        recs.append(e.recon())
        states.append(e.ltr_state() if ltr else None)
    return aus, recs, states, lts


def _assert_decodes(aus, recs, w, h):
    dec = avdec.decode_stream(aus, quiet=True)
    assert len(dec) == len(aus)
    for k, ((Y, U, V), (ry, ruv)) in enumerate(zip(dec, recs)):
        assert np.array_equal(Y, ry[:h, :w]), f"picture {k}: decoded luma != reconstruction"
        assert np.array_equal(U, ruv[:h // 2, 0:w:2]) and np.array_equal(V, ruv[:h // 2, 1:w:2]), f"picture {k}: chroma"


def _model_marks(frames, recs, pics, idrs):
    """the pictures the marking rule of tests/h264_model.py names, on its changed(k) from the source and picture k-1's reconstruction
    (an IDR counts every macroblock)"""
    h, w = recs[0][0].shape
    mbs = (w // 16) * (h // 16)
    out, prev = [], mbs
    for k, f in enumerate(frames):
        if k in idrs:
            prev = mbs
            continue
        y, _ = oracle.csc_nv12(f, coded_w=w, coded_h=h)
        changed = M.changed_count(y, recs[k - 1][0], pics[k].qp)
        if M.marks(changed, prev, mbs):
            out.append(k)
        prev = changed
    return out


def _check_syntax(frames, aus, recs, states, lts, idrs):
    pics = HSR.parse_stream(aus)
    marks = [k for k, p in enumerate(pics) if "mmco" in p.headers[0]]
    assert marks == [k for k, s in enumerate(states) if s["mark"]] == _model_marks(frames, recs, pics, set(idrs) | {0})
    for k, p in enumerate(pics):
        assert p.sps.max_num_ref_frames == 2 and p.sps.vui["max_dec_frame_buffering"] == 2
        for hd in p.headers:
            assert ("mmco" in hd) == (k in marks)
            if k in marks:
                assert hd["mmco"] == M.marking_ops(states[k]["active"]), (k, hd["mmco"])
            # the override exactly while a long-term picture exists
            assert hd.get("num_ref_idx_active", 1) == (2 if lts[k] is not None and not p.idr else 1), k
        if lts[k] is not None and not p.idr:
            # the model's DPB names the same long-term picture as the oracle's buffer holds
            assert len(p.ref_list) == 2 and p.ref_list[1] == pics[k - 1].long_term[0]
            assert np.array_equal(recs[p.ref_list[1]][0], lts[k][0]) and np.array_equal(recs[p.ref_list[1]][1], lts[k][1])
        for m in p.mbs:
            if m.ref_idx == 1:
                assert m.kind == "P_L0_16x16" and m.mv == (0, 0) and m.ref_pic == p.ref_list[1], (k, m.addr)
    return pics, marks


def _sad_checks(frames, pics, lts, qp, w, h):
    """every refIdx-1 macroblock's source block lies within the zero-motion threshold of the long-term picture at the zero vector"""
    thr = M.EARLY_SAD_PER_LAMBDA * M.LAMBDA[qp]
    cw, ch = (w + 15) & ~15, (h + 15) & ~15
    mbw = cw // 16
    n = 0
    for k, p in enumerate(pics):
        ones = [m for m in p.mbs if m.ref_idx == 1]
        if not ones:
            continue
        y, _ = oracle.csc_nv12(frames[k], coded_w=cw, coded_h=ch)
        for m in ones:
            r, c = divmod(m.addr, mbw)
            blk = y[16 * r: 16 * r + 16, 16 * c: 16 * c + 16].astype(int)
            lt = lts[k][0][16 * r: 16 * r + 16, 16 * c: 16 * c + 16].astype(int)
            assert np.abs(blk - lt).sum() <= thr, (k, m.addr)
            n += 1
    return n


@pytest.mark.parametrize("name", sorted(LC.CONTENTS))
@pytest.mark.parametrize("wide", [False, True])
def test_contents_decode_and_syntax(name, wide):
    w, h = 640, 368
    frames, _ = LC.CONTENTS[name](w, h)
    aus, recs, states, lts = _encode(frames, wide=wide, qp=26)
    _assert_decodes(aus, recs, w, h)
    pics, marks = _check_syntax(frames, aus, recs, states, lts, ())
    n = _sad_checks(frames, pics, lts, 26, w, h)
    if name in ("popup", "alt_tab"):
        assert marks and n > 0, (marks, n)
    for p in pics:
        assert not any(m.kind == "P_Skip" and m.ref_idx for m in p.mbs)


def test_cbr_idr_request_gop_and_paintover():
    """CBR with an IDR requested mid-stream (it clears the long-term picture) and a gop of 5 from picture 12 on; paint-over."""
    w, h = 640, 368
    frames = LC.popup(w, h)[0] + LC.alt_tab(w, h)[0]
    idrs = [8] + [k for k in range(12, len(frames)) if (k - 12) % 5 == 0]
    aus, recs, states, lts = _encode(frames, idr_at=idrs, paint=(3, 18, 2), rc_mode=0, target_bits=120000)
    _assert_decodes(aus, recs, w, h)
    _check_syntax(frames, aus, recs, states, lts, idrs)
    for k in idrs:
        assert lts[k + 1] is None if k + 1 < len(frames) else True      # an IDR retires the long-term picture


def test_resize_scaling_and_odd_cropped_size():
    """A resize is a fresh encoder (starting with an IDR); a scaled source and a cropped odd size decode as well."""
    for (sw, sh), (dw, dh) in (((640, 368), (640, 368)), ((800, 464), (800, 464)), ((1280, 720), (960, 544)), ((330, 202), (330, 202))):
        frames, _ = LC.popup(sw, sh)
        e = LongTermRefEncoder(dw, dh)
        e.set_long_term_ref(True)
        aus, recs = [], []
        for i, f in enumerate(frames):
            y, uv = oracle.csc_nv12(f, dst_w=dw, dst_h=dh, coded_w=e.cw, coded_h=e.ch)
            aus.append(e.encode_nv12(y, uv, i == 0, qp=28))
            recs.append(e.recon())
        _assert_decodes(aus, recs, dw, dh)
        assert any("mmco" in p.headers[0] for p in HSR.parse_stream(aus)), (sw, sh)


# Table A-1 MaxDpbMbs per level_idc
MAX_DPB_MBS = {31: 18000, 42: 34816, 51: 184320, 52: 184320, 62: 696320}


def test_two_reference_frames_fit_every_level():
    """max_num_ref_frames 2 <= MaxDpbFrames = min(MaxDpbMbs / (PicWidthInMbs * FrameHeightInMbs), 16) (A.3.1 h) at every size the
    encoder takes (16..7680 x 16..4320): the SPS the oracle writes, parsed by the syntax model."""
    sizes = [(w, h) for w in (16, 640, 1280, 1920, 2048, 2560, 3840, 4096, 5120, 7680) for h in (16, 480, 1080, 1440, 2160, 4320)]
    sizes += [(7680, 16), (16, 4320), (1920, 1088), (4096, 2304)]
    for w, h in sizes:
        e = LongTermRefEncoder(w, h)
        e.set_long_term_ref(True)
        sps = HS.parse_sps(HS.unescape(HS.split_annexb(e.encode_nv12(np.zeros((e.ch, e.cw), np.uint8), np.full((e.ch // 2, e.cw), 128, np.uint8), True))[0]))
        e.close()
        assert sps.max_num_ref_frames == 2 and sps.vui["max_dec_frame_buffering"] == 2
        assert min(MAX_DPB_MBS[sps.level_idc] // (sps.mbw * sps.mbh), 16) >= 2, (w, h, sps.level_idc)


# bytes of the pictures on which content comes back (640x368, CQP 26), measured with tools/long_term_ref_cost.py's rule at this size:
# the popup's closing picture and the first switch back to an application cost at most a fifth of their flag-off bytes.
RETURN_BOUND = 0.2


@pytest.mark.parametrize("name", ["popup", "alt_tab"])
def test_content_coming_back_is_cheap(name):
    w, h = 640, 368
    frames, returns = LC.CONTENTS[name](w, h)
    off = _encode(frames, ltr=False, qp=26)[0]
    on = _encode(frames, ltr=True, qp=26)[0]
    k = returns[0]
    assert len(on[k]) <= RETURN_BOUND * len(off[k]), (k, len(on[k]), len(off[k]))


@pytest.mark.parametrize("name", ["desktop", "predictor_paths", "noise", "gradient", "tiles"])
def test_no_regression_on_existing_contents(name):
    w, h = 640, 368
    frames = {
        "desktop": [synth.desktop(w, h, t) for t in range(8)],
        "predictor_paths": synth.predictor_paths(w, h),
        "noise": [synth.noise(w, h, s) for s in range(4)],
        "gradient": [synth.gradient(w, h, t) for t in range(8)],
        "tiles": [synth.tiles(w, h, noise_at=range(s, 920, 37), light_at=range(3 * s, 920, 11), seed=s) for s in range(6)],
    }[name]
    off = _encode(frames, ltr=False, qp=26)[0]
    on, recs, _, _ = _encode(frames, ltr=True, qp=26)
    _assert_decodes(on, recs, w, h)
    assert sum(map(len, on)) <= 1.02 * sum(map(len, off)), (sum(map(len, on)), sum(map(len, off)))


def test_flag_off_is_the_wide_oracle():
    """Without set_long_term_ref the encoder is exactly the oracle it extends."""
    from oracle.wide import WideRefEncoder
    frames = LC.popup(320, 192)[0]
    a = _encode(frames, ltr=False, qp=26)[0]
    e = WideRefEncoder(320, 192)
    assert a == [e.encode_bgra(f, i == 0, qp=26) for i, f in enumerate(frames)]


def test_reference_syntax_reader_agrees_on_single_reference_streams():
    """On a stream without the flag the extended reader returns what tests/h264_syntax.py does, every inter macroblock predicting
    from the picture just before."""
    frames = [synth.desktop(320, 192, t) for t in range(6)]
    aus = _encode(frames, ltr=False, qp=26)[0]
    for k, (a, b) in enumerate(zip(HS.parse_stream(aus), HSR.parse_stream(aus))):
        assert a.headers == b.headers and a.frame_num == b.frame_num and a.qp == b.qp
        for x, y in zip(a.mbs, b.mbs):
            assert (x.kind, x.mv, x.mvd, x.cbp, x.bits, x.skip_mv) == (y.kind, y.mv, y.mvd, y.cbp, y.bits, y.skip_mv)
            assert x.luma is None and y.luma is None or np.array_equal(x.luma, y.luma)
            assert y.ref_idx == 0 and (y.intra or y.ref_pic == k - 1)

