"""Droppable pictures (B2V_FLAG_DROPPABLE) in the oracle, checked against the H.264 syntax model and libavcodec: the layer pattern,
the frame_num rule and the unchanged SPS; the full stream decodes to the oracle's reconstruction of every picture and the stream
without its non-reference access units to the reconstruction of every picture kept; a dropped REFERENCE picture does not (the
check can fail).  Also the one-byte test a consumer applies and the RTC mailbox's drop policy."""
import asyncio

import numpy as np
import pytest

import oracle
from oracle import avdec
from oracle.layers import LayeredRefEncoder
from selkies_b200.h264_nal import is_droppable
from selkies_b200.rtc_bridge import PipelineBridge, VideoSample
from tests import h264_syntax as HS
from tests import synth

W, H = 320, 192


def _idrs(n, idr_at=(), gop=-1):
    """The IDR decision of b2v_api.cu for n pictures: a request before each index in idr_at, `gop` pictures per IDR when > 0."""
    out, since = [], 0
    for i in range(n):
        idr = i == 0 or i in idr_at or (gop > 0 and since >= gop)
        since = 1 if idr else since + 1
        out.append(idr)
    return out


def _encode(frames, droppable=True, idr_at=(), gop=-1, w=W, h=H, **kw):
    """(access units, reconstruction (Y, UV) after every picture, IDR flags)."""
    e = LayeredRefEncoder(w, h)
    e.set_droppable(droppable)
    idrs = _idrs(len(frames), idr_at, gop)
    aus, recs = [], []
    for f, idr in zip(frames, idrs):
        aus.append(e.encode_bgra(f, idr, **kw))
        recs.append(e.recon())
    return aus, recs, idrs


def _slice_ref_idc(au):
    """nal_ref_idc of every slice NAL of an access unit."""
    return [n[0] >> 5 & 3 for n in HS.split_annexb(au) if n[0] & 31 in (1, 5)]


def _assert_decodes_to(aus, recs, w, h):
    dec = avdec.decode_stream(aus, quiet=True)
    assert len(dec) == len(aus), f"{len(dec)} pictures decoded of {len(aus)}"
    for k, ((Y, U, V), (ry, ruv)) in enumerate(zip(dec, recs)):
        assert np.array_equal(Y, ry[:h, :w]), f"picture {k}: decoded luma != reconstruction"
        assert np.array_equal(U, ruv[:h // 2, 0:w:2]) and np.array_equal(V, ruv[:h // 2, 1:w:2]), f"picture {k}: chroma"


def _check_stream(aus, recs, idrs, w=W, h=H):
    # syntax: every access unit parses under the model, slices agree on nal_ref_idc, the layer pattern restarts at each IDR
    pics = HS.parse_stream(aus)
    fn, since, prev_ref = 0, 0, True
    for k, (au, pic, idr) in enumerate(zip(aus, pics, idrs)):
        idcs = set(_slice_ref_idc(au))
        assert len(idcs) == 1, f"picture {k}: slices disagree on nal_ref_idc {idcs}"
        idc = idcs.pop()
        if idr:
            since, fn = 0, 0
        assert pic.idr == idr
        want = 3 if idr else (0 if since % 2 else 2)
        assert idc == want, f"picture {k} (count {since} from the IDR): nal_ref_idc {idc}, expected {want}"
        assert prev_ref or idc, f"picture {k}: two non-reference pictures in a row"
        assert pic.frame_num == fn, f"picture {k}: frame_num {pic.frame_num}, expected {fn}"
        assert is_droppable(au) == (idc == 0)
        if idc:
            fn = (fn + 1) % 256
        prev_ref, since = idc != 0, since + 1
    # the whole stream decodes to the reconstruction of every picture
    _assert_decodes_to(aus, recs, w, h)
    # ... and so does the stream without its non-reference access units, to the reconstruction of every picture kept
    keep = [k for k, au in enumerate(aus) if not is_droppable(au)]
    assert len(keep) < len(aus)
    _assert_decodes_to([aus[k] for k in keep], [recs[k] for k in keep], w, h)


def test_sps_is_the_flag_off_sps():
    f = synth.desktop(W, H, 0)
    on, _, _ = _encode([f], True, rc_mode=1, qp=26)
    off, _, _ = _encode([f], False, rc_mode=1, qp=26)
    sps = lambda au: [n for n in HS.split_annexb(au) if n[0] & 31 in (7, 8)]
    assert sps(on[0]) == sps(off[0]) and len(sps(on[0])) == 2
    assert on[0] == off[0]                      # the IDR picture itself is coded as without the flag


@pytest.mark.parametrize("qp", [0, 26, 51])
def test_desktop_scroll(qp):
    frames = [synth.desktop(W, H, t) for t in range(10)]
    _check_stream(*_encode(frames, rc_mode=1, qp=qp))


def test_predictor_paths():
    _check_stream(*_encode(synth.predictor_paths(W, H), rc_mode=1, qp=28))


def test_noise_and_gradient_pan():
    frames = [synth.noise(W, H, s) for s in range(3)] + [synth.gradient(W, H, t) for t in range(8)]
    _check_stream(*_encode(frames, rc_mode=1, qp=30))


@pytest.mark.parametrize("rc", ["cqp", "cbr"])
def test_idr_request_and_gop_restart_the_pattern(rc):
    """An IDR requested at an odd count (after a non-reference picture) and then a gop of 5: the pattern restarts each time."""
    kw = dict(rc_mode=1, qp=27) if rc == "cqp" else dict(rc_mode=0, target_bits=60000)
    frames = [synth.desktop(W, H, t) for t in range(21)]
    aus, recs, idrs = _encode(frames, idr_at=(4,), gop=5, **kw)
    assert [k for k, i in enumerate(idrs) if i] == [0, 4, 9, 14, 19]
    _check_stream(aus, recs, idrs)


def test_cropped_picture():
    w, h = 328, 200
    frames = [synth.desktop(w, h, t) for t in range(7)]
    _check_stream(*_encode(frames, w=w, h=h, rc_mode=1, qp=24), w=w, h=h)


def test_layered_stream_differs_from_the_flag_off_stream():
    """The flag changes the P pictures (reference and predictor); with it off the stream is the flag-off stream."""
    frames = [synth.desktop(W, H, t) for t in range(6)]
    on, _, _ = _encode(frames, True, rc_mode=1, qp=26)
    off, _, _ = _encode(frames, False, rc_mode=1, qp=26)
    assert on[0] == off[0] and on[2:] != off[2:]
    assert not any(is_droppable(a) for a in off)


def test_dropping_a_reference_picture_corrupts_until_the_next_idr():
    """Control: the check above can fail.  Without reference P picture 4 every later picture up to the next IDR decodes wrong."""
    frames = [synth.desktop(W, H, t) for t in range(12)]
    aus, recs, idrs = _encode(frames, idr_at=(9,), rc_mode=1, qp=26)
    assert not is_droppable(aus[4]) and idrs[9]
    keep = [k for k in range(len(aus)) if k != 4]
    dec = avdec.decode_stream([aus[k] for k in keep], quiet=True)
    assert len(dec) == len(keep)
    same = {k: np.array_equal(d[0], recs[k][0][:H, :W]) for d, k in zip(dec, keep)}
    assert all(same[k] for k in (0, 1, 2, 3))
    assert not any(same[k] for k in (5, 6, 7, 8)), same
    assert all(same[k] for k in (9, 10, 11))


def test_oracle_refuses_stripes_with_droppable():
    e = LayeredRefEncoder(W, 256)
    e.set_droppable(True)
    with pytest.raises(ValueError):
        e.set_stripes(4)
    e2 = LayeredRefEncoder(W, 256)
    e2.set_stripes(4)
    with pytest.raises(ValueError):
        e2.set_droppable(True)
    e2.set_droppable(False)
    e3 = LayeredRefEncoder(W, 256)
    e3.set_droppable(True)
    assert e3.set_stripes(16) == 1                # as many rows as the picture: full frame, allowed


def test_is_droppable_reads_the_first_slice_header():
    assert is_droppable(b"\x00\x00\x00\x01\x01\x88")
    assert not is_droppable(b"\x00\x00\x00\x01\x41\x88")
    assert not is_droppable(b"\x00\x00\x00\x01\x67\x42\x00\x00\x01\x68\xce\x00\x00\x01\x65\x88")   # IDR behind SPS/PPS
    assert is_droppable(b"\x04\x00\x00\x01\x00\x00\x01\x40\x00\x40\x00\x00\x00\x01\x01\x9a", 10)   # behind a 10-byte header
    assert not is_droppable(b"") and not is_droppable(b"\xff\xd8\xff\xe0") and not is_droppable(b"\x00\x00\x01")


class _S:
    def __init__(self, name, droppable=None):
        self.name = name
        if droppable is not None:
            self.droppable = droppable


def test_mailbox_sheds_droppable_samples_first():
    async def run():
        b = PipelineBridge()
        await b.set_data(_S("r0", False))
        await b.set_data(_S("d1", True))         # a reference waits: the new droppable sample goes
        assert b.dropped == 1 and b.dropped_reference == 0
        await b.set_data(_S("r2", False))        # two references: the older goes, and is counted
        assert b.dropped == 2 and b.dropped_reference == 1
        assert (await b.get_data()).name == "r2"
        await b.set_data(_S("d3", True))
        await b.set_data(_S("r4", False))        # a droppable sample waits: it goes
        assert b.dropped == 3 and b.dropped_reference == 1
        await b.set_data(_S("x5"))               # no attribute: a reference
        assert b.dropped == 4 and b.dropped_reference == 2
        assert (await b.get_data()).name == "x5"
        await b.set_data(_S("d6", True))
        await b.set_data(_S("d7", True))         # droppable after droppable: the older goes
        assert b.dropped == 5 and b.dropped_reference == 2
        assert (await b.get_data()).name == "d7"
    asyncio.run(run())


def test_mailbox_keeps_an_oracle_stream_decodable():
    """A consumer at half the encoder's rate: the mailbox sheds only the non-reference pictures, and what the consumer takes
    decodes to the encoder's reconstructions."""
    frames = [synth.desktop(W, H, t) for t in range(13)]
    aus, recs, _ = _encode(frames, rc_mode=1, qp=26)
    samples = [VideoSample(a, k) for k, a in enumerate(aus)]
    assert [s.droppable for s in samples] == [False] + [k % 2 == 1 for k in range(1, 13)]

    async def run():
        b, got = PipelineBridge(), []
        for k, s in enumerate(samples):
            await b.set_data(s)
            if k % 2 == 0:
                got.append(await b.get_data())
        return b, got
    b, got = asyncio.run(run())
    assert b.dropped_reference == 0 and b.dropped == 6
    kept = [s.pts for s in got]
    assert kept == [0, 2, 4, 6, 8, 10, 12]
    _assert_decodes_to([aus[k] for k in kept], [recs[k] for k in kept], W, H)


@pytest.mark.parametrize("mode", ["jpeg", "striped"])
def test_screen_capture_refuses_droppable_outside_full_frame_h264(mode):
    """Refused before any session exists (the library refuses the same combinations: tests/test_droppable_gpu.py)."""
    from selkies_b200.pixelflux_compat import CaptureSettings, ScreenCapture
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height = 640, 384
    cs.h264_droppable_frames = True
    if mode == "jpeg":
        cs.output_mode = 0
    else:
        cs.h264_fullframe = False
    with pytest.raises(ValueError, match="h264_droppable_frames"):
        ScreenCapture().start_capture(cs, lambda *a: None)


def test_media_pipeline_sets_droppable_frames():
    from selkies_b200.media_pipeline import MediaPipelineB200
    loop = asyncio.new_event_loop()
    try:
        assert MediaPipelineB200(loop, droppable_frames=True).generate_capture_settings().h264_droppable_frames is True
        assert MediaPipelineB200(loop).generate_capture_settings().h264_droppable_frames is False
    finally:
        loop.close()
