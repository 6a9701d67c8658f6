"""Scene cuts (B2V_FLAG_SCENE_CUT) in the oracle.  On every pair of the scene-cut table at QP 26 and 36 the rule picks the smaller
picture; on the scripted contents of tests/ltr_content.py and tests/wide_content.py, with wide motion, droppable pictures and the
long-term reference on and off, in CQP and in CBR with an IDR request, a gop and paint-over, every stream decodes with libavcodec to
the oracle's reconstructions after every picture and costs at most 1 % more than with the flag off.  The independent reader of
tests/h264_syntax.py finds every cut picture as NAL type 1 whose slices are all of slice_type 7, in the IDR slice grid, frame_num
continuous, and the SPS byte-identical to the flag-off stream's."""
import numpy as np
import pytest

import oracle
from oracle import RefEncoder, avdec
from oracle.scut import SceneCutEncoder
from tests import h264_syntax as HS
from tests import h264_syntax_refs as HSR
from tests import ltr_content as LC
from tests import scut_scenario as SC
from tests import synth
from tests import wide_content as WC

W, H = 1920, 1080


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def _pairs(w, h):
    return {
        "desktop_inverted": (LC.desktop(w, h, 1), LC.desktop(w, h, 1, invert=True)),
        "desktop_bars": (synth.desktop(w, h), synth.bars(w, h)),
        "desktop_gradient": (synth.desktop(w, h), synth.gradient(w, h)),
        "gradient_desktop": (synth.gradient(w, h), synth.desktop(w, h)),
        "desktop_desktop": (synth.desktop(w, h, seed=1), synth.desktop(w, h, seed=2)),
        "noise_noise": (synth.noise(w, h, 0), synth.noise(w, h, 1)),
    }


def _encode(frames, cut=True, wide=False, ltr=False, droppable=False, w=None, h=None, idr_at=(), paint=None, **kw):
    h_, w_ = frames[0].shape[:2]
    e = SceneCutEncoder(w or w_, h or h_)
    if paint:
        e.set_paintover(*paint)
    e.set_droppable(droppable)
    e.set_wide_motion(wide)
    e.set_long_term_ref(ltr)
    e.set_scene_cut(cut)
    aus, recs, cuts = [], [], []
    for i, f in enumerate(frames):
        aus.append(e.encode_bgra(f, i == 0 or i in idr_at, **kw))
        recs.append(e.recon())
        cuts.append(bool(cut and e.scut_state()["cut"]))
    e.close()
    return aus, recs, cuts


def _assert_decodes(aus, recs, w, h):
    dec = avdec.decode_stream(aus, quiet=True)
    assert len(dec) == len(aus)
    for k, ((Y, U, V), (ry, ruv)) in enumerate(zip(dec, recs)):
        assert np.array_equal(Y, ry[:h, :w]), f"picture {k}: decoded luma != reconstruction"
        assert np.array_equal(U, ruv[:h // 2, 0:w:2]) and np.array_equal(V, ruv[:h // 2, 1:w:2]), f"picture {k}: chroma"


@pytest.mark.parametrize("qp", [26, 36])
def test_pairs_pick_the_smaller_picture(qp):
    for name, (a, b) in _pairs(W, H).items():
        p_aus, _, _ = _encode([a, b], cut=False, qp=qp)
        aus, recs, cuts = _encode([a, b], qp=qp)
        e = RefEncoder(W, H)
        intra = len(e.encode_bgra(b, True, qp=qp))          # the second picture as an IDR picture
        e.close()
        assert cuts[1] == (intra < len(p_aus[1])), (name, qp, cuts[1], intra, len(p_aus[1]))
        assert len(aus[1]) <= len(p_aus[1]), name
        if name in ("desktop_inverted", "desktop_bars", "desktop_gradient"):
            assert 5 * len(aus[1]) <= len(p_aus[1]), (name, len(aus[1]), len(p_aus[1]))
        _assert_decodes(aus, recs, W, H)


def _scripts(w, h):
    out = {k: f(w, h)[0] for k, f in LC.CONTENTS.items() if k in ("popup", "alt_tab", "drag", "scroll")}
    out["wide_scroll"] = [WC.desktop_scroll(w, h, t, 24) for t in range(6)]
    out["wide_drag"] = [WC.drag(w, h, t, (40, 16), (100, 100)) for t in range(6)]
    out["switches"] = SC.switches(w, h)
    return out


@pytest.mark.parametrize("mode", ["plain", "wide", "ltr", "wide_ltr", "droppable"])
def test_scripts_decode_and_cost_no_more(mode):
    kw = dict(wide="wide" in mode, ltr="ltr" in mode, droppable=mode == "droppable")
    w, h = 1280, 720
    for name, frames in _scripts(w, h).items():
        for qp in (26, 36):
            off, _, _ = _encode(frames, cut=False, qp=qp, **kw)
            aus, recs, cuts = _encode(frames, qp=qp, **kw)
            _assert_decodes(aus, recs, w, h)
            assert sum(map(len, aus)) <= 1.01 * sum(map(len, off)), (mode, name, qp)
            if name == "switches":
                assert cuts[2] and not cuts[1] and not cuts[3], (mode, qp, cuts)


def test_cbr_idr_request_gop_and_paintover():
    w, h = 640, 368
    frames = SC.switches(w, h) + LC.alt_tab(w, h)[0]
    aus, recs, cuts = _encode(frames, idr_at=(8, 16, 21), paint=(3, 18, 2), rc_mode=0, target_bits=6_000_000 // 60)
    _assert_decodes(aus, recs, w, h)
    assert any(cuts)


def test_syntax_of_cut_pictures():
    """NAL type 1, every slice an I slice in the IDR grid (one row, idr_slice_mbs columns), frame_num continuous, SPS unchanged."""
    w, h = 1280, 720
    frames = SC.switches(w, h)
    off, _, _ = _encode(frames, cut=False)
    aus, recs, cuts = _encode(frames)
    assert aus[0] == off[0]                              # the IDR, SPS and PPS included, is byte-identical
    pics = HS.parse_stream(aus)
    idr_slices = len(HS.parse_stream(aus[:1])[0].headers)
    for k, (au, p) in enumerate(zip(aus, pics)):
        types = [n[0] & 0x1F for n in HS.split_annexb(au) if n[0] & 0x1F in (1, 5)]
        if k == 0:
            continue
        assert p.frame_num == k % 256 and not p.idr and set(types) == {1}, k
        kinds = {hd["slice_type"] for hd in p.headers}
        assert kinds == ({2} if cuts[k] else {0}), (k, kinds, cuts[k])
        if cuts[k]:
            assert len(p.headers) == idr_slices and all(n[0] & 0x1F != 7 for n in HS.split_annexb(au)), k
    assert [k for k in range(len(aus)) if cuts[k]] == [k for k, p in enumerate(pics) if k and p.headers[0]["slice_type"] == 2]


def test_long_term_ref_and_droppable_syntax():
    """With the long-term reference the cut pictures keep the P picture's marking; with droppable pictures its nal_ref_idc."""
    w, h = 640, 368
    frames = SC.switches(w, h) + LC.alt_tab(w, h)[0]
    aus, recs, cuts = _encode(frames, ltr=True)
    pics = HSR.parse_stream(aus)
    assert any(cuts) and all(p.sps.max_num_ref_frames == 2 for p in pics)
    aus, recs, cuts = _encode(frames, droppable=True)
    pics = HS.parse_stream(aus)
    for k, p in enumerate(pics):
        assert p.nal_ref_idc == (0 if k % 2 else (3 if k == 0 else 2)), k
    _assert_decodes(aus, recs, w, h)


@pytest.mark.parametrize("qp", [26, 36])
def test_returning_content_stays_p_under_long_term_ref(qp):
    """The long-term picture's zero vector is every macroblock's candidate in cost_inter: the closing popup and the switch back to an
    application, which it predicts, stay P pictures (the switch away is cut)."""
    w, h = 1280, 720
    for name in ("popup", "alt_tab"):
        frames, returns = LC.CONTENTS[name](w, h)
        _, _, cuts = _encode(frames, ltr=True, qp=qp)
        assert returns and not any(cuts[k] for k in returns), (name, qp, returns, cuts)
        assert any(cuts), (name, qp)


@pytest.mark.parametrize("mode", ["plain", "wide", "ltr", "wide_ltr", "droppable"])
def test_nothing_cut_is_the_flag_off_stream(mode):
    """Where no picture is cut (scroll, drag), the access units and reconstructions are byte-identical to the flag-off stream's: the
    P analysis, the slices and the rate control run unchanged."""
    kw = dict(wide="wide" in mode, ltr="ltr" in mode, droppable=mode == "droppable")
    w, h = 640, 368
    for frames in (LC.scroll(w, h)[0], LC.drag(w, h)[0], [WC.desktop_scroll(w, h, t, 24) for t in range(6)]):
        for qp in (26, 36):
            off, roff, _ = _encode(frames, cut=False, qp=qp, **kw)
            on, ron, cuts = _encode(frames, qp=qp, **kw)
            assert not any(cuts), (mode, qp, cuts)
            assert on == off, (mode, qp)
            assert all(np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) for a, b in zip(roff, ron)), (mode, qp)
