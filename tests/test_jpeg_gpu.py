"""GPU parity of the JPEG stripe mode (CaptureSettings.output_mode = 0; B2V_FLAG_JPEG) through the C-ABI: every delivered stripe
must be, byte for byte, the JFIF file oracle/jpeg_ref.c makes of the same rows (JFIF colour conversion by oracle/csc_ref.c),
and libjpeg-turbo must decode it."""
import numpy as np
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import synth

pytestmark = pytest.mark.gpu
cv2 = pytest.importorskip("cv2")


def run(w, h, frames, quality=60, stripe_rows=0, header=N.B2V_HDR_NONE, **kw):
    with Session(w, h, flags=N.B2V_FLAG_JPEG, rc_mode=N.B2V_RC_CQP, crf=quality, stripe_rows=stripe_rows, header_mode=header, **kw) as s:
        for f in frames:
            s.submit(f)
            s.flush()
        return s.take_frames()


def stripe_rows_of(h, stripe_rows):
    mcu_h = (h + 15) // 16
    return stripe_rows if 0 < stripe_rows < mcu_h else (stripe_rows and mcu_h) or (mcu_h + 7) // 8


# 640x96 in one stripe: at quality 92 its FF bytes sit at the last byte of a thread's 16-byte chunk and past the first 4096-byte
# round of the stuffing copy (test_escape_cases_oracle.py checks that it reaches both)
@pytest.mark.parametrize("w,h,stripe_rows", [(64, 48, 0), (320, 192, 3), (130, 70, 2), (640, 362, 0), (1920, 1080, 0), (640, 96, 6)])
@pytest.mark.parametrize("quality", [1, 35, 60, 92, 100])
def test_jpeg_stripes_bit_exact(w, h, stripe_rows, quality):
    f = synth.desktop(w, h, 1) if w >= 128 else synth.noise(w, h, 1)
    got = run(w, h, [f], quality, stripe_rows)
    rows = stripe_rows_of(h, stripe_rows) * 16
    assert len(got) == -(-h // rows)                     # first picture: every stripe
    canvas = np.zeros((h, w, 3), np.uint8)
    for k, g in enumerate(got):
        y0 = k * rows
        assert (g.y_start, g.height, g.frame_id) == (y0, min(rows, h - y0), 0)
        ref = oracle.jpeg_encode_bgra(np.ascontiguousarray(f[y0: y0 + rows]), quality)
        assert g.data == ref, f"stripe {k}: first difference at byte {next((i for i in range(min(len(ref), len(g.data))) if ref[i] != g.data[i]), -1)} of {len(ref)} / {len(g.data)}"
        dec = cv2.imdecode(np.frombuffer(g.data, np.uint8), cv2.IMREAD_COLOR)
        assert dec is not None and dec.shape[:2] == (g.height, w)
        canvas[y0: y0 + g.height] = dec
    if quality >= 60 and w >= 128:                       # (the 64x48 case is pure noise)
        mse = np.mean((canvas.astype(float) - f[..., :3].astype(float)) ** 2)
        assert 10 * np.log10(255 ** 2 / max(mse, 1e-9)) > 22.0


def test_jpeg_only_changed_stripes_and_paintover():
    """Damage detection at stripe granularity + paint-over: a stripe static for `trigger` pictures is sent once more at the
    paint-over quality (CaptureSettings.paint_over_jpeg_quality / paint_over_trigger_frames)."""
    w, h, rows = 320, 192, 3            # 12 MCU rows -> 4 stripes of 48 rows
    a = synth.desktop(w, h, 0)
    b = a.copy()
    b[100:110, 40:80, :3] = (10, 200, 30)                 # touches stripe 2 only (rows 96..143)
    frames = [a, a, b, b, b, b, b]
    got = run(w, h, frames, 50, rows, paintover_trigger_frames=2, paintover_crf=95)
    by_frame = {}
    for g in got:
        by_frame.setdefault(g.frame_id, []).append(g)
    assert [g.y_start for g in by_frame[0]] == [0, 48, 96, 144]
    assert 1 not in by_frame                               # nothing changed
    # picture 2: the damaged stripe at the normal quality; stripes 0, 1, 3 have now been static for two pictures -> repainted at 95
    assert [g.y_start for g in by_frame[2]] == [0, 48, 96, 144]
    for g in by_frame[2]:
        src, q = (b, 50) if g.y_start == 96 else (a, 95)
        assert g.data == oracle.jpeg_encode_bgra(np.ascontiguousarray(src[g.y_start: g.y_start + 48]), q), g.y_start
    assert 3 not in by_frame
    # stripe 2 is repainted two unchanged pictures after its change; after that nothing is sent any more
    assert [g.y_start for g in by_frame[4]] == [96] and by_frame[4][0].data == oracle.jpeg_encode_bgra(np.ascontiguousarray(b[96:144]), 95)
    assert 5 not in by_frame and 6 not in by_frame


def test_jpeg_pixelflux_header_and_screen_capture():
    """ScreenCapture(output_mode=0): the callback sees frame_id u16be | y_start u16be | JFIF (selkies.py:3116-3118 adds 03 00)."""
    import threading
    from selkies_b200.pixelflux_compat import ArraySource, CaptureSettings, ScreenCapture
    w, h = 320, 192
    frames = [synth.desktop(w, h, t) for t in range(3)]
    got, done = [], threading.Event()

    def cb(ptr, _u):
        r = ptr.contents
        got.append(bytes(r.data[:r.size]))
        if len(got) >= 8:
            done.set()
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.target_fps, cs.output_mode, cs.jpeg_quality = w, h, 120.0, 0, 70
    cap = ScreenCapture(ArraySource(frames, loop=False))
    cap.start_capture(cs, cb)
    done.wait(10)
    cap.stop_capture()
    assert len(got) >= 8
    rows = ((h // 16 + 7) // 8) * 16
    first = [g for g in got if int.from_bytes(g[0:2], "big") == 0]
    assert len(first) == -(-h // rows)
    for g in first:
        y0 = int.from_bytes(g[2:4], "big")
        assert g[4:6] == b"\xff\xd8" and g[4:] == oracle.jpeg_encode_bgra(np.ascontiguousarray(frames[0][y0: y0 + rows]), 70)
