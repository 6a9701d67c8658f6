"""GPU parity, striped mode ("x264enc-striped", CaptureSettings.h264_fullframe = False, selkies.py:3219): the CUDA encoder's
stripes vs oracle/h264_ref.c, bit-exact, through the C-ABI (tests/scenario.py); every stripe stream decodes on its own (libavcodec)."""
import numpy as np
import pytest

from oracle import avdec
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import scenario as S
from tests import synth

pytestmark = pytest.mark.gpu


def frames_with_static_top(w, h, n):
    frames = [synth.desktop(w, h, t) for t in range(n)]
    for f in frames[1:]:
        f[:64] = frames[0][:64]
    return frames


def encode(w, h, frames, stripe_rows, slice_rows, idr_at=(), **cfg):
    """Both encoders over `frames` in striped mode; returns the oracle's Expected records."""
    cfg = S.Config(w, h, stripe_rows=stripe_rows, slice_rows=slice_rows, **cfg)
    return S.pictures(S.run(cfg, S.stream(frames, idr_at)))


@pytest.mark.parametrize("w,h,stripe_rows,slice_rows", [(320, 200, 4, 1), (320, 200, 4, 2), (320, 200, 6, 3), (192, 112, 1, 1), (640, 360, 8, 1), (320, 200, 4, 0), (640, 360, 6, 0)])
def test_stripes_bit_exact(w, h, stripe_rows, slice_rows):
    """Every band's bytes, height and key flag; every band's stream decodes on its own (checked by the driver)."""
    xs = encode(w, h, frames_with_static_top(w, h, 5), stripe_rows, slice_rows, idr_at=(3,))
    assert [x.is_key for x in xs] == [True, False, False, True, False]
    if (w, stripe_rows) == (320, 4):
        assert all(y0 >= 64 for y0, _ in xs[1].bands)          # the static band is not sent


def test_stripes_subpel_motion_stays_inside_the_band():
    """A vertical pan: vectors that would leave the band see the band's edge padding instead, exactly as each band's decoder does."""
    cv2 = pytest.importorskip("cv2")
    w, h, rows = 320, 192, 3
    rng = np.random.default_rng(7)
    big = cv2.GaussianBlur(rng.normal(0, 1, (h + 96, w + 96, 3)).astype(np.float32), (0, 0), 4) * 700 + 128
    frames = []
    for t in range(4):
        a = cv2.warpAffine(big, np.float32([[1, 0, -(24 + 0.75 * t)], [0, 1, -(24 + 3.25 * t)]]), (w, h), flags=cv2.INTER_CUBIC)
        frames.append(np.dstack([np.clip(a, 0, 255).astype(np.uint8), np.full((h, w), 255, np.uint8)]))
    encode(w, h, frames, rows, 1, qp=26)


def test_stripes_cbr_and_pixelflux_header():
    w, h, rows = 320, 200, 4
    xs = encode(w, h, frames_with_static_top(w, h, 8), rows, 1, rc_mode=S.CBR, kbps=900, fps=30.0, header_mode=S.HDR_PIXELFLUX)
    assert [x.is_key for x in xs] == [True] + [False] * 7 and len({x.qp for x in xs}) > 1


def test_stripe_rows_must_be_a_multiple_of_slice_rows():
    with pytest.raises(Exception):
        Session(320, 200, rc_mode=N.B2V_RC_CQP, crf=28, slice_rows=2, stripe_rows=3).close()


def test_screen_capture_striped_mode():
    """CaptureSettings.h264_fullframe = False -> stripes with the 10-byte header, one decoder per y_start (selkies-ws-core.js:3183-3216)."""
    import threading
    from selkies_b200.pixelflux_compat import ArraySource, CaptureSettings, ScreenCapture
    w, h = 320, 200
    frames = frames_with_static_top(w, h, 6)
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.target_fps = w, h, 120.0
    cs.h264_fullframe, cs.h264_crf, cs.h264_stripe_rows = False, 28, 4
    seen, done = [], threading.Event()

    def cb(result_ptr, _):
        r = result_ptr.contents
        seen.append(bytes(r.data[:r.size]))
        if int.from_bytes(seen[-1][2:4], "big") >= 5 and int.from_bytes(seen[-1][4:6], "big") == 192:
            done.set()

    cap = ScreenCapture(ArraySource(frames, loop=False))
    cap.start_capture(cs, cb)
    assert done.wait(20)
    cap.stop_capture()
    by_y = {}
    for d in seen:
        assert d[0] == 0x04
        by_y.setdefault(int.from_bytes(d[4:6], "big"), []).append(d[10:])
    assert sorted(by_y) == [0, 64, 128, 192]
    assert len(by_y[0]) == 1 and len(by_y[64]) == 6          # static top stripe: key frame only
    for y0, st in by_y.items():
        Y, _, _ = avdec.decode_stream(st, quiet=True)[-1]
        assert Y.shape == (min(h, y0 + 64) - y0, w)


def test_ws_video_channel_carries_stripes_from_the_native_thread():
    """ScreenCapture (striped) -> WsVideoChannel.on_stripe on the native output thread -> sender task -> per-stripe decoders."""
    import asyncio
    from selkies_b200.pixelflux_compat import ArraySource, CaptureSettings, ScreenCapture, StripeCallback
    from selkies_b200.ws_video import WsVideoChannel
    w, h = 320, 200
    frames = frames_with_static_top(w, h, 6)

    async def run():
        loop = asyncio.get_running_loop()
        sent = []

        async def send(b):
            sent.append(b)
        ch = WsVideoChannel(send, loop, queue_depth=256, fps=120.0)
        sender = asyncio.ensure_future(ch.run_sender())
        cs = CaptureSettings()
        cs.capture_width, cs.capture_height, cs.target_fps = w, h, 120.0
        cs.h264_fullframe, cs.h264_crf, cs.h264_stripe_rows = False, 28, 4
        cap = ScreenCapture(ArraySource(frames, loop=False))
        await loop.run_in_executor(None, cap.start_capture, cs, StripeCallback(ch.on_stripe))
        for _ in range(400):
            await asyncio.sleep(0.01)
            if ch.last_sent_id >= 5 and ch.queue.empty():
                break
        await loop.run_in_executor(None, cap.stop_capture)
        await asyncio.sleep(0.05)
        await ch.queue.join()
        sender.cancel()
        ch.on_ack(f"CLIENT_FRAME_ACK {ch.last_sent_id}")
        assert ch.evaluate_gate() and ch.dropped == 0
        return sent
    sent = asyncio.run(run())
    by_y = {}
    for d in sent:
        assert d[0] == 0x04
        by_y.setdefault(int.from_bytes(d[4:6], "big"), []).append(d[10:])
    assert sorted(by_y) == [0, 64, 128, 192] and len(by_y[0]) == 1
    for y0, st in by_y.items():
        Y, _, _ = avdec.decode_stream(st, quiet=True)[-1]
        assert Y.shape == (min(h, y0 + 64) - y0, w)
