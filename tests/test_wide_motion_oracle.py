"""Wide-range motion (B2V_FLAG_WIDE_MOTION) in the oracle: fast scrolls and window drags are coded as motion.  Every stream decodes with
libavcodec to the oracle's reconstructions; the macroblocks parsed by the syntax model carry the true displacement; P pictures of a fast
scroll cost a fraction of the flag-off bytes; no vector leaves the range the SPS asserts, droppable streams included; the flag costs
the existing contents at most 2 %; and with the flag off the oracle's bytes are those it always produced."""
import numpy as np
import pytest

import oracle
from oracle import avdec
from oracle.wide import WideRefEncoder
from tests import h264_syntax as HS
from tests import synth
from tests import wide_content as WC

MV_LIMIT = 1023            # quarter samples: the SPS's VUI log2_max_mv_length_horizontal / vertical = 10


@pytest.fixture(scope="module", autouse=True)
def _threads():
    oracle.set_threads(0)


def _encode(frames, wide=True, w=None, h=None, droppable=False, stripes=0, **kw):
    h_, w_ = frames[0].shape[:2]
    w, h = w or w_, h or h_
    e = WideRefEncoder(w, h)
    if stripes:
        e.set_stripes(stripes)
    e.set_droppable(droppable)
    e.set_wide_motion(wide)
    aus, recs = [], []
    for i, f in enumerate(frames):
        aus.append(e.encode_bgra(f, i == 0, **kw))
        recs.append(e.recon())
    return aus, recs


def _assert_decodes(aus, recs, w, h):
    dec = avdec.decode_stream(aus, quiet=True)
    assert len(dec) == len(aus)
    for k, ((Y, U, V), (ry, ruv)) in enumerate(zip(dec, recs)):
        assert np.array_equal(Y, ry[:h, :w]), f"picture {k}: decoded luma != reconstruction"
        assert np.array_equal(U, ruv[:h // 2, 0:w:2]) and np.array_equal(V, ruv[:h // 2, 1:w:2]), f"picture {k}: chroma"


def _mv_share(pic, mbs, mv, w):
    """Share of the macroblocks (mbx, mby) coded as P_Skip or P_L0_16x16 with vector `mv` (quarter samples)."""
    mbw = (w + 15) // 16
    hit = sum(1 for (x, y) in mbs if pic.mbs[y * mbw + x].kind in ("P_Skip", "P_L0_16x16") and tuple(pic.mbs[y * mbw + x].mv) == mv)
    return hit / len(mbs)


def _max_mv(pics):
    return max((max(abs(m.mv[0]), abs(m.mv[1])) for p in pics for m in p.mbs if not m.intra), default=0)


# ---- scrolls: from a still picture (the motion starts in picture 2) and in steady state -------------------------------------
W, H = 1920, 1080


@pytest.mark.parametrize("speed", [17, 24, 40, 64, 128, 250])
def test_scroll_vectors_and_decode(speed):
    frames = [WC.desktop_scroll(W, H, 0, speed)] * 2 + [WC.desktop_scroll(W, H, t, speed) for t in range(1, 6)]
    aus, recs = _encode(frames)
    _assert_decodes(aus, recs, W, H)
    pics = HS.parse_stream(aus)
    mbs = WC.interior_mbs(WC.scroll_region(W, H, speed), W, H)
    for k in range(2, 7):          # 2: the first moving picture (no temporal predictor), then steady state
        share = _mv_share(pics[k], mbs, (0, 4 * speed), W)
        assert share >= 0.9, f"picture {k}: {share:.3f} of {len(mbs)} macroblocks carry (0, {4 * speed})"
    assert _max_mv(pics) <= MV_LIMIT


@pytest.mark.parametrize("v", [(40, -30), (-100, 0), (127, 60)])
def test_drag_vectors_and_decode(v):
    w, h = 1280, 720
    start = (560 - 2 * v[0], 240 - 2 * v[1])
    frames = [WC.drag(w, h, 0, v, start)] * 2 + [WC.drag(w, h, t, v, start) for t in range(1, 5)]
    aus, recs = _encode(frames)
    _assert_decodes(aus, recs, w, h)
    pics = HS.parse_stream(aus)
    for k in range(2, 6):
        # two macroblocks in from the window's edges: a group that straddles an edge may take its anchor's background vector
        mbs = WC.interior_mbs(WC.drag_window_at(k - 1, v, start), w, h, margin=2)
        share = _mv_share(pics[k], mbs, (-4 * v[0], -4 * v[1]), w)
        assert share >= 0.9, f"picture {k}: {share:.3f} of {len(mbs)} window macroblocks carry {(-4 * v[0], -4 * v[1])}"
    assert _max_mv(pics) <= MV_LIMIT


def test_motion_at_picture_and_band_edges():
    """A window dragged into the corner of a small picture, and a scroll in a striped session whose bands clamp the coarse search:
    the streams decode, and every band of the striped one decodes to its rows of the reconstruction."""
    w, h = 336, 208
    frames = [WC.drag(w, h, t, (-37, -29), (150, 100), 160, 112) for t in range(7)]
    aus, recs = _encode(frames)
    _assert_decodes(aus, recs, w, h)
    assert _max_mv(HS.parse_stream(aus)) <= MV_LIMIT
    w, h, rows = 640, 480, 8
    frames = [WC.desktop_scroll(w, h, t, 40) for t in range(6)]
    e = WideRefEncoder(w, h)
    e.set_stripes(rows)
    e.set_wide_motion(True)
    bands = {}
    for i, f in enumerate(frames):
        au = e.encode_bgra(f, i == 0)
        ry, _ = e.recon()
        for b, (o, sz, coded) in enumerate(e.stripe_table()):
            if coded:
                bands.setdefault(b, []).append((au[o:o + sz], ry[b * rows * 16:(b + 1) * rows * 16].copy()))
    for b, items in bands.items():
        dec = avdec.decode_stream([a for a, _ in items], quiet=True)
        for (Y, _, _), (_, ref) in zip(dec, items):
            assert np.array_equal(Y, ref[:Y.shape[0], :w]), f"band {b}"


# ---- bytes --------------------------------------------------------------------------------------------------------------------
def _p_bytes(speed, wide):
    aus, _ = _encode([WC.desktop_scroll(W, H, t, speed) for t in range(6)], wide=wide)
    return int(np.mean([len(a) for a in aus[2:6]]))


# bytes per P picture (pictures 2..5) with the flag off: 1080p, CQP 26, the desktop's text region scrolled
FLAG_OFF = {8: 15184, 16: 28528, 24: 575833, 40: 713988, 96: 576276}


@pytest.mark.parametrize("speed", sorted(FLAG_OFF))
def test_flag_off_bytes_unchanged(speed):
    assert _p_bytes(speed, False) == FLAG_OFF[speed]


@pytest.mark.parametrize("speed", [24, 40, 64])
def test_fast_scroll_bytes(speed):
    off = FLAG_OFF.get(speed) or _p_bytes(speed, False)
    on = _p_bytes(speed, True)
    assert on * 5 <= off, f"{speed} px: {on} bytes per P picture with the flag, {off} without"


def test_droppable_vector_range():
    """Droppable streams double the temporal predictor of a picture two back: a 128 px scroll predicts 256 px, outside the range —
    the candidate is refused and no coded vector leaves [-1023, 1023]."""
    w, h = 1280, 720
    for speed in (100, 128, 200):
        frames = [WC.desktop_scroll(w, h, t, speed) for t in range(8)]
        aus, recs = _encode(frames, droppable=True)
        _assert_decodes(aus, recs, w, h)
        assert _max_mv(HS.parse_stream(aus)) <= MV_LIMIT


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
    off, _ = _encode(frames, wide=False)
    on, recs = _encode(frames, wide=True)
    _assert_decodes(on, recs, w, h)
    assert sum(map(len, on)) <= 1.02 * sum(map(len, off)), (sum(map(len, on)), sum(map(len, off)))
