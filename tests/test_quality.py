"""CPU side of B2V_FLAG_QUALITY: the numpy statement of the measurement (tests/quality_ref.py) against two independent float64
forms of SSIM, its record geometry, the C ABI's layout and argument errors, and the Python conversion.  No GPU needed."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

from tests import quality_ref as Q

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pair(rng, h, w, spread):
    s = rng.integers(0, 256, (h, w), dtype=np.uint8)
    r = np.clip(s.astype(np.int64) + rng.integers(-spread, spread + 1, (h, w)), 0, 255).astype(np.uint8)
    return s, r


@pytest.mark.parametrize("h,w", [(8, 8), (12, 8), (8, 14), (16, 16), (18, 22), (30, 34), (36, 20)])
@pytest.mark.parametrize("spread", [0, 3, 40, 255])
def test_statement_equals_direct_per_window_ssim(h, w, spread):
    rng = np.random.default_rng(h * 1000 + w * 10 + spread)
    s, r = _pair(rng, h, w, spread)
    got, ref = Q.ssim_windows(s, r), Q.ssim_direct(s, r)
    assert got.shape == ref.shape == ((h - 8) // 4 + 1, (w - 8) // 4 + 1)
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-12)
    if spread == 0:
        assert np.all(got == 1.0)


def test_statement_extremes():
    """Black against white, flat against noise, and a negatively correlated window: every value in [-1, 1] and as the direct
    form says."""
    rng = np.random.default_rng(5)
    noise = rng.integers(0, 256, (16, 16), dtype=np.uint8)
    cases = [(np.zeros((16, 16), np.uint8), np.full((16, 16), 255, np.uint8)),
             (np.full((16, 16), 128, np.uint8), noise),
             (noise, (255 - noise).astype(np.uint8))]
    for s, r in cases:
        got = Q.ssim_windows(s, r)
        np.testing.assert_allclose(got, Q.ssim_direct(s, r), rtol=0, atol=1e-12)
        assert np.all(np.abs(got) <= 1.0)
    assert np.all(Q.ssim_windows(noise, 255 - noise) < 0)


@pytest.mark.parametrize("h,w,spread", [(256, 384, 6), (270, 482, 60), (64, 1920, 1)])
def test_statement_equals_box_filter_ssim(h, w, spread):
    rng = np.random.default_rng(h + w)
    s, r = _pair(rng, h, w, spread)
    got, ref = Q.ssim_windows(s, r), Q.ssim_boxfilter(s, r)
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=0, atol=1e-9)
    assert abs(got.mean() - ref.mean()) < 1e-12


def _nv12(rng, cw, ch):
    return rng.integers(0, 256, (ch, cw), dtype=np.uint8), rng.integers(0, 256, (ch // 2, cw), dtype=np.uint8)


def test_measure_counts_the_record_only():
    """Rows outside the record and columns at or beyond dst_w (the coded padding) never count; Cb is the even byte of a chroma
    pair, Cr the odd one."""
    rng = np.random.default_rng(9)
    cw, ch, dst_w = 144, 96, 130
    sy, suv = _nv12(rng, cw, ch)
    ry, ruv = sy.copy(), suv.copy()
    ry[:, dst_w:] ^= 0xFF                       # padding columns: ignored
    ruv[:, dst_w:] ^= 0xFF
    ry[10, 5] = sy[10, 5] ^ 1                   # in the band at 0
    ry[40, 7] = sy[40, 7] ^ 3                   # in the band at 32
    ruv[20, 8] = suv[20, 8] ^ 2                 # Cb, luma row 40
    ruv[20, 9] = suv[20, 9] ^ 4                 # Cr, luma row 40
    top, mid = Q.measure(sy, suv, ry, ruv, dst_w, 0, 32), Q.measure(sy, suv, ry, ruv, dst_w, 32, 32)
    d = lambda a, b: (int(a) - int(b)) ** 2
    assert (top["sse_y"], top["sse_cb"], top["sse_cr"]) == (d(sy[10, 5], ry[10, 5]), 0, 0)
    assert (mid["sse_y"], mid["sse_cb"], mid["sse_cr"]) == (d(sy[40, 7], ry[40, 7]), d(suv[20, 8], ruv[20, 8]), d(suv[20, 9], ruv[20, 9]))
    assert (mid["samples_y"], mid["samples_c"]) == (130 * 32, 130 * 32 // 4)
    # windows: origins x = 0, 4, .., 120 (x + 8 <= 130) and y = 32, 36, .., 56 (y + 8 <= 64)
    assert mid["ssim_windows"] == 31 * 7
    short = Q.measure(sy, suv, ry, ruv, dst_w, 90, 6)
    assert short["ssim_windows"] == 0 and math.isnan(short["ssim_y"])


def test_b2v_quality_layout_matches_header():
    from selkies_b200 import _native as N
    src = open(os.path.join(ROOT, "include", "b2video.h")).read()
    body = re.search(r"typedef struct b2v_quality \{(.*?)\} b2v_quality;", src, re.S).group(1)
    fields = []
    for ctype, names in re.findall(r"(int64_t|double)\s+([^;]+);", body):
        fields += [(n.strip(), ctype) for n in names.split(",")]
    ctypes_of = {"int64_t": C.c_int64, "double": C.c_double}
    assert [(n, ctypes_of[t]) for n, t in fields] == [(n, t) for n, t in N.B2VQuality._fields_]
    assert C.sizeof(N.B2VQuality) == 56 and N.B2VQuality.ssim_y.offset == 40
    assert int(re.search(r"B2V_FLAG_QUALITY\s*=\s*(\d+)", src).group(1)) == N.B2V_FLAG_QUALITY == 64


def test_frame_quality_argument_and_state_errors():
    """No CUDA call is reached: null arguments are B2V_EINVAL, a handle whose callback is not running on this thread B2V_ESTATE
    (the handle is never dereferenced)."""
    from selkies_b200 import _native as N
    lib = N.lib()
    q = N.B2VQuality()
    assert lib.b2v_frame_quality(None, C.byref(q)) == N.B2V_EINVAL
    assert lib.b2v_frame_quality(None, None) == N.B2V_EINVAL
    fake = C.c_void_p(0x1000)
    assert lib.b2v_frame_quality(fake, None) == N.B2V_EINVAL
    assert lib.b2v_frame_quality(fake, C.byref(q)) == N.B2V_ESTATE
    assert b"callback" in lib.b2v_last_error()


@pytest.mark.parametrize("other", ["B2V_FLAG_JPEG", "B2V_FLAG_NO_ENCODE"])
def test_create_rejects_quality_without_a_reconstruction(other):
    from selkies_b200 import _native as N
    lib = N.lib()
    s = N.B2VSettings()
    s.src_w, s.src_h, s.fps, s.flags = 320, 192, 60.0, N.B2V_FLAG_QUALITY | getattr(N, other)
    h = C.c_void_p()
    assert lib.b2v_create(C.byref(s), N.FRAME_CB(lambda f, u: None), None, C.byref(h)) == N.B2V_EINVAL
    assert other.encode() in lib.b2v_last_error()


def test_frame_quality_conversion():
    from selkies_b200 import _native as N
    from selkies_b200.session import FrameQuality
    q = N.B2VQuality(sse_y=1000, sse_cb=0, sse_cr=10, samples_y=640, samples_c=160, ssim_y=0.75, ssim_windows=12)
    fq = FrameQuality.from_native(q)
    assert fq.sse == (1000, 0, 10) and fq.samples == (640, 160) and fq.ssim == 0.75
    assert fq.psnr[0] == pytest.approx(10 * math.log10(255 ** 2 * 640 / 1000)) and fq.psnr[1] == math.inf
    assert fq.psnr[2] == pytest.approx(10 * math.log10(255 ** 2 * 160 / 10))
    q.ssim_y, q.ssim_windows = float("nan"), 0
    assert FrameQuality.from_native(q).ssim is None


def test_capture_settings_quality_metrics_defaults_off():
    from selkies_b200.pixelflux_compat import CaptureSettings
    assert CaptureSettings().quality_metrics is False
