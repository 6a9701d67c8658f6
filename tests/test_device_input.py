"""CPU: the checks of device-frame ingest that need no GPU.  b2v_submit_device's argument errors that return before any CUDA
call, the Python reading of `__cuda_array_interface__` (hand-built interfaces: no device memory behind them), and how
ScreenCapture hands a DeviceFrameSource's window to the session."""
import ctypes as C
import subprocess
import sys

import numpy as np
import pytest

from selkies_b200 import _native as N
from selkies_b200.pixelflux_compat import ArraySource, DeviceFrameSource, ScreenCapture
from selkies_b200.session import PIXEL_FORMATS, device_frame_args


class Cai:
    """An object exposing a hand-built __cuda_array_interface__."""

    def __init__(self, shape, typestr="|u1", strides=None, ptr=0x7f0000000000, **extra):
        self.__cuda_array_interface__ = dict(shape=shape, typestr=typestr, strides=strides, data=(ptr, False), version=3 if extra else 2,
                                             **extra)


def test_c_abi_argument_errors_before_any_cuda_call():
    lib = N.lib()
    for fmt in (-1, 4, 99):
        assert lib.b2v_submit_device(None, 0x1000, 1280, fmt, None, 0) == N.B2V_EINVAL
        assert b"unknown pixel format" in lib.b2v_last_error()
    assert lib.b2v_submit_device(None, 0x1000, 1280, N.B2V_PIX_RGB, None, 0) == N.B2V_EINVAL
    assert b"null" in lib.b2v_last_error()
    buf = C.create_string_buffer(64)
    assert lib.b2v_submit_device(C.c_void_p(1), None, 1280, N.B2V_PIX_BGRA, None, 0) == N.B2V_EINVAL    # null frame
    assert lib.b2v_submit_device(None, C.addressof(buf), 1280, N.B2V_PIX_BGRA, None, 0) == N.B2V_EINVAL  # null handle


def test_pixel_format_codes_match_the_header():
    assert {k: v[0] for k, v in PIXEL_FORMATS.items()} == {"BGRA": 0, "RGBA": 1, "BGR": 2, "RGB": 3}
    assert {k: v[1] for k, v in PIXEL_FORMATS.items()} == {"BGRA": 4, "RGBA": 4, "BGR": 3, "RGB": 3}


def test_window_pointer_pitch_and_format():
    base = 0x7f0000000000
    ptr, pitch, fmt, st = device_frame_args(Cai((100, 200, 4), ptr=base), 200, 100, 0)
    assert (ptr, pitch, fmt, st) == (base, 800, N.B2V_PIX_BGRA, 0)
    ptr, pitch, fmt, _ = device_frame_args(Cai((120, 260, 3), strides=(1024, 3, 1), ptr=base), 200, 100, 0, "RGB", origin=(7, 11))
    assert (ptr, pitch, fmt) == (base + 11 * 1024 + 7 * 3, 1024, N.B2V_PIX_RGB)
    ptr, _, fmt, _ = device_frame_args(Cai((100, 201, 4), ptr=base), 200, 100, 0, "RGBA", origin=(1, 0))
    assert (ptr, fmt) == (base + 4, N.B2V_PIX_RGBA)


def test_stream_rules():
    f = Cai((10, 20, 4))
    assert device_frame_args(f, 20, 10, 0)[3] == 0                               # nothing said: the legacy default stream
    assert device_frame_args(f, 20, 10, 0, stream=0xabc)[3] == 0xabc              # an explicit handle
    assert device_frame_args(f, 20, 10, 0, stream=type("S", (), {"cuda_stream": 0xdef})())[3] == 0xdef
    for cai_stream, handle in ((None, 0), (1, 1), (2, 2), (0x1234, 0x1234)):       # version 3: None / legacy / per-thread / handle
        assert device_frame_args(Cai((10, 20, 4), stream=cai_stream), 20, 10, 0)[3] == handle
    assert device_frame_args(Cai((10, 20, 4), stream=0x1234), 20, 10, 0, stream=0x99)[3] == 0x99    # explicit wins


@pytest.mark.parametrize("frame,fmt,origin,exc", [
    (Cai((10, 20, 4), typestr="<u2"), "BGRA", (0, 0), TypeError),                   # dtype
    (Cai((10, 20, 4), typestr="<f4"), "BGRA", (0, 0), TypeError),
    (Cai((10, 20, 3)), "BGRA", (0, 0), ValueError),                                  # shape does not match the format
    (Cai((10, 20, 4)), "RGB", (0, 0), ValueError),
    (Cai((10, 80)), "BGRA", (0, 0), ValueError),                                     # 2-D
    (Cai((10, 20, 4), strides=(160, 8, 1)), "BGRA", (0, 0), ValueError),             # pixels not packed
    (Cai((10, 20, 4), strides=(80, 4, 2)), "BGRA", (0, 0), ValueError),
    (Cai((10, 20, 4), strides=(4, 40, 1)), "BGRA", (0, 0), ValueError),              # column-major rows
    (Cai((10, 20, 4)), "BGRA", (1, 0), ValueError),                                  # window outside the array
    (Cai((10, 20, 4)), "BGRA", (0, 1), ValueError),
    (Cai((10, 20, 4)), "BGRA", (-1, 0), ValueError),
    (Cai((10, 20, 4)), "YUYV", (0, 0), ValueError),                                  # unknown format
    (np.zeros((10, 20, 4), np.uint8), "BGRA", (0, 0), TypeError),                    # host array
])
def test_rejected_before_the_c_call(frame, fmt, origin, exc):
    with pytest.raises(exc):
        device_frame_args(frame, 20, 10, 0, fmt, origin)


def test_product_does_not_import_torch():
    code = ("import sys, selkies_b200.session, selkies_b200.pixelflux_compat, selkies_b200.media_pipeline; "
            "assert 'torch' not in sys.modules, 'torch imported'")
    subprocess.check_call([sys.executable, "-c", code])


class _FakeSession:
    def __init__(self):
        self.calls = []

    def submit_device(self, frame, **kw):
        self.calls.append(("device", frame, kw))

    def acquire(self):
        return 0, np.zeros((4, 8, 4), np.uint8)

    def submit_slot(self, slot, capture_ns=0):
        self.calls.append(("ring", slot))


def test_screen_capture_hands_the_capture_window_to_submit_device():
    class Src(DeviceFrameSource):
        pixel_format, stream = "RGB", 0x55

        def frame(self, index):
            return None if index >= 2 else f"surface{index}"
    cs = ScreenCapture(Src())
    cs._origin = (37, 150)
    fake = _FakeSession()
    assert cs._encode_next(fake, 0) and cs._encode_next(fake, 1) and not cs._encode_next(fake, 2)
    assert [c[1] for c in fake.calls] == ["surface0", "surface1"]
    kw = fake.calls[0][2]
    assert (kw["pixel_format"], kw["stream"], kw["origin"]) == ("RGB", 0x55, (37, 150))


def test_host_sources_ignore_the_capture_origin():
    cs = ScreenCapture(ArraySource([np.full((4, 8, 4), 9, np.uint8)]))
    cs._origin = (37, 150)
    fake = _FakeSession()
    assert cs._encode_next(fake, 0)
    assert fake.calls == [("ring", 0)]
