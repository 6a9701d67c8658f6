"""GPU tests of the reference-facing Python surface: pixelflux-compatible ScreenCapture, MediaPipelineB200
(mirror of MediaPipelinePixel) and the GSTWebRTCApp façade — end to end on the CUDA pipeline."""
import asyncio
import threading
import time

import numpy as np
import pytest

import oracle
from oracle import avdec
from selkies_b200.gst_webrtc_app import GSTWebRTCApp, GSTWebRTCAppError
from selkies_b200.media_pipeline import MediaPipelineB200, RateControlMode
from selkies_b200.pixelflux_compat import ArraySource, CaptureSettings, ScreenCapture, StripeCallback
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import scenario as S
from tests import synth
from tests.test_h264_oracle import split_nals

pytestmark = pytest.mark.gpu


def wait_for(pred, timeout=20.0):
    t0 = time.time()
    while not pred():
        if time.time() - t0 > timeout:
            raise TimeoutError
        time.sleep(0.01)


def test_screen_capture_contract_and_parity():
    w, h = 320, 192
    frames = [synth.desktop(w, h, t) for t in range(6)]
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.target_fps = w, h, 200.0
    cs.output_mode, cs.h264_cbr_mode, cs.h264_crf = 1, False, 28
    got, threads = [], set()

    def cb(result_ptr, user):
        if not result_ptr:
            return
        r = result_ptr.contents
        threads.add(threading.get_ident())
        got.append((r.frame_id, bytes(r.data[10:r.size]), bytes(r.data[:r.size])))   # both reference idioms

    cap = ScreenCapture(ArraySource(frames, loop=False))
    cap.start_capture(cs, StripeCallback(cb))
    wait_for(lambda: len(got) >= len(frames))
    cap.stop_capture()
    assert threading.get_ident() not in threads                 # fired on the native output thread
    assert [g[0] for g in got[:6]] == list(range(6))            # frame_id +1 per frame (pts derives from it)
    enc = oracle.RefEncoder(w, h)
    for i, f in enumerate(frames):
        ref = enc.encode_bgra(f, i == 0, qp=28)
        assert got[i][1] == ref                                  # same bytes as the oracle behind the plugin API
        hdr = got[i][2][:10]
        assert hdr[0] == 0x04 and hdr[1] == (1 if i == 0 else 0) and int.from_bytes(hdr[2:4], "big") == i
    with pytest.warns(RuntimeWarning):                           # h264_fullcolor: accepted, the stream stays 4:2:0 (superset decoder config)
        fc = CaptureSettings()
        fc.capture_width, fc.capture_height, fc.h264_fullcolor = 64, 48, True
        cap2 = ScreenCapture(ArraySource([synth.noise(64, 48, 1)], loop=False))
        cap2.start_capture(fc, lambda p, u: None)
        cap2.stop_capture()


def test_media_pipeline_b200_end_to_end():
    w, h = 320, 192

    async def scenario():
        loop = asyncio.get_running_loop()
        out = []
        p = MediaPipelineB200(loop, "x264enc", framerate=120, video_bitrate=2, width=w, height=h, rc_mode=RateControlMode.CBR,
                              frame_source=ArraySource([synth.desktop(w, h, t) for t in range(8)]))

        async def produce(buf, pts, kind):
            out.append((buf, pts, kind))
        p.produce_data = produce
        await p.start_media_pipeline()
        assert p.is_media_pipeline_running()
        while len(out) < 10:
            await asyncio.sleep(0.01)
        await p.set_video_bitrate(4)
        await p.set_framerate(60)
        n = len(out)
        await p.dynamic_idr_frame()
        while len(out) < n + 8:
            await asyncio.sleep(0.01)
        await p.stop_media_pipeline()
        assert not p.is_media_pipeline_running()
        return out

    out = asyncio.run(scenario())
    assert all(k == "video" for _, _, k in out)
    assert out[0][0][:5] == b"\x00\x00\x00\x01\x67"              # first AU: SPS (in-band, rtc.py:394-401)
    keys = [i for i, (b, _, _) in enumerate(out) if (split_nals(b)[0][0] & 31) == 7]
    assert keys[0] == 0 and len(keys) >= 2                       # the requested IDR arrived
    assert out[1][1] - out[0][1] == 90000 // 120                 # pts step (media_pipeline.py:291-292)
    dec = avdec.decode_stream([b for b, _, _ in out], quiet=True)
    assert len(dec) == len(out) and dec[0][0].shape == (h, w)


def test_gst_webrtc_app_facade():
    w, h = 256, 144
    app = GSTWebRTCApp(framerate=200, video_bitrate=1500, width=w, height=h, frame_source=ArraySource([synth.bars(w, h, t) for t in range(8)]))
    samples = []
    app.on_video_sample = lambda data, pts, key: samples.append((data, pts, key))
    with pytest.raises(GSTWebRTCAppError):
        app.set_framerate(30)                                     # pipeline not built yet
    app.build_video_pipeline()
    wait_for(lambda: len(samples) >= 5)
    app.set_video_bitrate(3000)
    app.set_framerate(100)
    n = len(samples)
    app.set_resolution(320, 180)                                  # 180 -> coded 192, cropped
    wait_for(lambda: len(samples) >= n + 6)
    app.send_idr()
    app.stop_pipeline()
    assert samples[0][2] is True
    # after the resize: new SPS/PPS + IDR, and the stream decodes at the new size
    idx = next(i for i in range(1, len(samples)) if samples[i][2])
    dec = avdec.decode_stream([s[0] for s in samples[idx:]], quiet=True)
    assert dec and dec[0][0].shape == (180, 320)
    dec0 = avdec.decode_stream([s[0] for s in samples[:idx]], quiet=True)
    assert dec0[0][0].shape == (h, w)


def test_scaled_encode_matches_oracle():
    S.run(S.Config(640, 360, 320, 180, qp=29), [S.picture(synth.desktop(640, 360, t)) for t in range(3)])


def test_two_concurrent_sessions_are_independent():
    """The reference keeps one capture instance per display (selkies.py:3178-3181): two sessions driven from two threads
    on the same GPU must each produce exactly the stream a lone session produces."""
    import threading
    from selkies_b200 import _native as N
    from selkies_b200.session import Session
    cfgs = [(320, 192, 28, [synth.desktop(320, 192, t) for t in range(6)]), (256, 144, 33, [synth.bars(256, 144, t) for t in range(6)])]
    solo = []
    for w, h, qp, frames in cfgs:
        with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=qp) as s:
            for f in frames:
                s.submit(f)
            s.flush()
            solo.append([g.data for g in s.take_frames()])
    out = [None, None]

    def worker(i):
        w, h, qp, frames = cfgs[i]
        with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=qp) as s:
            for f in frames:
                s.submit(f)
                s.set_bitrate_kbps(5000 + i)          # control calls racing with submits must be harmless
            s.flush()
            out[i] = [g.data for g in s.take_frames()]

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=120)
    assert out[0] == solo[0] and out[1] == solo[1]


def test_ring_release_returns_a_slot_without_encoding():
    """b2v_ring_release: the producer acquired a slot and then had no frame; the next acquire hands out the same slot and the
    stream continues as if nothing happened (frame ids stay consecutive)."""
    w, h = 128, 96
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=30, ring_slots=3) as s:
        s.submit(synth.desktop(w, h, 0))
        slot, view = s.acquire()
        s.release_slot(slot)
        with pytest.raises(Exception):
            s.release_slot(slot)                      # already free
        slot2, view2 = s.acquire()
        assert slot2 == slot
        view2[...] = synth.desktop(w, h, 1)
        s.submit_slot(slot2)
        s.flush()
        got = s.take_frames()
    assert [g.frame_id for g in got] == [0, 1] and got[0].is_key and not got[1].is_key


def test_finite_source_ends_without_a_stale_frame():
    from selkies_b200.pixelflux_compat import ArraySource, CaptureSettings, ScreenCapture
    w, h = 128, 96
    frames = [synth.desktop(w, h, t) for t in range(5)]
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.target_fps, cs.h264_crf = w, h, 240.0, 30
    seen = []
    cap = ScreenCapture(ArraySource(frames, loop=False))
    cap.start_capture(cs, lambda p, u: seen.append(p.contents.frame_id))
    cap._thread.join(10)                              # the capture thread stops by itself when the source is exhausted
    cap.stop_capture()
    assert seen == [0, 1, 2, 3, 4]
