"""B2V_FLAG_QUALITY on the GPU: every delivered record's measurement equals the numpy statement (tests/quality_ref.py) applied to
the oracle's NV12 of the picture and the oracle's reconstruction after it, which the GPU equals bit for bit: SSEs exactly, SSIM
to within 1e-9.  The access units must still equal the oracle's, and the flag must not change a byte of them."""
import ctypes
import dataclasses
import math
import threading
import time

import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.session import Session
from tests import quality_ref as Q
from tests import scenario as S
from tests import synth
from tests import tensor_scenario as T

pytestmark = pytest.mark.gpu


def run_quality(cfg: S.Config, events, side=S.GpuSide) -> list:
    """Applies `events` to the oracle and to a GPU session with B2V_FLAG_QUALITY; checks every delivered record (bytes, frame id,
    y_start, height, quality) against the oracle and the statement.  Returns the GPU's records."""
    cfg = dataclasses.replace(cfg, flags=cfg.flags | N.B2V_FLAG_QUALITY)
    o, g = S.OracleSide(cfg), side(cfg)
    expected = []
    try:
        for ev in events:
            if ev[0] != "picture":
                o.control(ev)
                g.control(ev)
                continue
            x = o.picture(ev[1], "")
            e = o.enc
            sy, suv = oracle.csc_nv12(ev[1], o.dst[0], o.dst[1], e.cw, e.ch)
            ry, ruv = e.recon()
            w, h = o.dst
            for y0, au in x.bands:
                bh = S._band_height(cfg, h, y0)
                expected.append((x.index, y0, bh, au, Q.measure(sy, suv, ry, ruv, w, y0, bh)))
            g.picture(ev[1])
        g.s.flush()
        got = g.s.take_frames()
    finally:
        g.s.close()
    assert len(got) == len(expected), f"{len(got)} records delivered, the oracle codes {len(expected)}"
    for f, (idx, y0, bh, au, m) in zip(got, expected):
        where = f"picture {idx}, band y_start {y0}"
        assert (f.frame_id, f.y_start, f.height) == (idx, y0, bh), where
        assert f.data == au, f"{where}: access unit differs from the oracle's"
        q = f.quality
        assert q is not None, where
        assert q.sse == (m["sse_y"], m["sse_cb"], m["sse_cr"]), f"{where}: sse {q.sse}, statement {(m['sse_y'], m['sse_cb'], m['sse_cr'])}"
        assert q.samples == (m["samples_y"], m["samples_c"]), where
        if m["ssim_windows"] == 0:
            assert q.ssim is None, f"{where}: ssim {q.ssim} without windows"
        else:
            assert q.ssim is not None and abs(q.ssim - m["ssim_y"]) <= 1e-9, f"{where}: ssim {q.ssim}, statement {m['ssim_y']}"
    return got


def desktop(w, h, n, t0=0):
    return [synth.desktop(w, h, t0 + t) for t in range(n)]


@pytest.mark.parametrize("qp", [0, 26, 51])
def test_cqp(qp):
    got = run_quality(S.Config(320, 192, qp=qp), S.stream(desktop(320, 192, 5)))
    if qp == 51:
        assert all(f.quality.sse[0] > 0 for f in got)


def test_cbr_with_mid_stream_idr():
    frames = desktop(352, 208, 8)
    got = run_quality(S.Config(352, 208, rc_mode=S.CBR, kbps=1500, fps=30.0), S.stream(frames, idr_at=(5,)))
    assert [f.is_key for f in got] == [True] + [False] * 4 + [True] + [False] * 2


def test_noise_at_qp0_is_lossless():
    """Noise at QP 0 is coded as I_PCM: the reconstruction is the source."""
    frames = [synth.noise(256, 144, s) for s in range(3)]
    for f in run_quality(S.Config(256, 144, qp=0), S.stream(frames)):
        assert f.quality.sse == (0, 0, 0) and f.quality.psnr == (math.inf,) * 3 and f.quality.ssim == 1.0


def test_cropped_size():
    run_quality(S.Config(130, 70, qp=30), S.stream(desktop(130, 70, 4)))


def test_scaled_session():
    run_quality(S.Config(320, 192, dst_width=202, dst_height=118, qp=24), S.stream(desktop(320, 192, 4)))


def test_striped_4k():
    run_quality(S.Config(3840, 2160, qp=28, stripe_rows=17), S.stream(desktop(3840, 2160, 3)))


def test_last_band_under_8_rows():
    """Bands of 32 rows over 100 rows: the last band holds 4 visible rows and no SSIM window."""
    frames = [synth.bars(192, 100, t) for t in range(3)]
    got = run_quality(S.Config(192, 100, qp=26, stripe_rows=2), S.stream(frames))
    last = [f for f in got if f.y_start == 96]
    assert last and all(f.height == 4 and f.quality.ssim is None for f in last)


def test_resize_mid_stream():
    ev = S.stream(desktop(320, 192, 3)) + [S.resize(256, 160)] + S.stream(desktop(256, 160, 3, 3)) + \
        [S.resize(320, 192, 160, 96)] + S.stream(desktop(320, 192, 2, 6))
    run_quality(S.Config(320, 192, qp=27), ev)


def test_tensor_stream():
    cfg = T.TensorConfig(320, 192, qp=26, dtype="f16")
    run_quality(cfg, T.tensorise(cfg, S.stream(desktop(320, 192, 4))), side=T.TensorGpuSide)


def test_headline_4k():
    """bench.py's configuration: 4K CBR 20 Mbit/s, resident frames, the 16-picture scroll cycle and its restart."""
    oracle.set_threads(0)
    frames = [synth.desktop(3840, 2160, t) for t in range(16)]
    cfg = S.Config(3840, 2160, rc_mode=S.CBR, kbps=20000, fps=60.0, ring_slots=16, flags=N.B2V_FLAG_TIMING_CSC, entry="resident")
    run_quality(cfg, [S.picture(frames[i % 16]) for i in range(18)])


def _encode(quality: bool, frames, **kw):
    with Session(320, 192, rc_mode=N.B2V_RC_CQP, crf=26, quality=quality, **kw) as s:
        for f in frames:
            s.submit(f)
        s.flush()
        return [f.data for f in s.take_frames()], s.stats()["kernel_launches"]


@pytest.mark.parametrize("stripe_rows", [0, 4])
def test_flag_changes_no_byte_and_adds_one_launch_per_picture(stripe_rows):
    frames = desktop(320, 192, 6)
    off, n_off = _encode(False, frames, stripe_rows=stripe_rows)
    on, n_on = _encode(True, frames, stripe_rows=stripe_rows)
    assert on == off
    assert n_on - n_off == len(frames)


def test_state_errors():
    lib = N.lib()
    q = N.B2VQuality()
    for quality, want in ((True, N.B2V_OK), (False, N.B2V_ESTATE)):
        holder, seen = [], []
        with Session(320, 192, collect=False, quality=quality,
                     on_frame=lambda fptr: seen.append(lib.b2v_frame_quality(holder[0]._h, ctypes.byref(q)))) as s:
            holder.append(s)
            assert lib.b2v_frame_quality(s._h, ctypes.byref(q)) == N.B2V_ESTATE        # outside a callback
            s.submit(synth.desktop(320, 192, 0))
            s.flush()
        assert seen == [want], (quality, seen)                                          # ESTATE: no B2V_FLAG_QUALITY
    for flags in (N.B2V_FLAG_JPEG, N.B2V_FLAG_NO_ENCODE):
        with pytest.raises(N.B2VError) as e:
            Session(320, 192, flags=flags, quality=True)
        assert e.value.code == N.B2V_EINVAL


def test_screen_capture_quality_metrics():
    from selkies_b200.pixelflux_compat import ArraySource, CaptureSettings, ScreenCapture
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.target_fps, cs.h264_crf = 320, 192, 120.0, 30
    cs.quality_metrics = True
    got, done = [], threading.Event()

    def cb(res, _user):
        got.append(res.contents.quality)
        if len(got) >= 4:
            done.set()

    cap = ScreenCapture(ArraySource(desktop(320, 192, 4)))
    cap.start_capture(cs, cb)
    done.wait(30)
    cap.stop_capture()
    assert len(got) >= 4
    for q in got:
        assert q is not None and q.samples == (320 * 192, 320 * 192 // 4)
        assert 0.5 < q.ssim <= 1.0 and all(p > 25 for p in q.psnr)
    cs.quality_metrics = False
    plain = []
    cap = ScreenCapture(ArraySource(desktop(320, 192, 2)))
    cap.start_capture(cs, lambda res, u: plain.append(res.contents.quality))
    t0 = time.time()
    while not plain and time.time() - t0 < 30:
        time.sleep(0.01)
    cap.stop_capture()
    assert plain and all(q is None for q in plain)
