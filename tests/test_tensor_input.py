"""CPU: the checks of tensor ingest that need no GPU.  b2v_submit_tensor's argument errors that return before any CUDA call, the
layout of b2v_tensor, the Python reading of `__cuda_array_interface__` (hand-built interfaces: no device memory behind them),
and how ScreenCapture tells a TensorFrameSource from a DeviceFrameSource."""
import ctypes as C
import os
import re
import sys
import types

import numpy as np
import pytest

from selkies_b200 import _native as N
from selkies_b200.pixelflux_compat import DeviceFrameSource, ScreenCapture, TensorFrameSource
from selkies_b200.session import DTYPES, tensor_frame_args
from tests.test_device_input import Cai, _FakeSession

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = 0x7f0000000000


def _tensor(data=0x1000, dtype=N.B2V_DT_F16, fmt=N.B2V_PIX_RGB, sc=4096, sy=64, sx=2):
    return N.B2VTensor(data, dtype, fmt, sc, sy, sx)


@pytest.mark.parametrize("entry", ["b2v_submit_tensor", "b2v_csc_nv12_tensor"])
def test_c_abi_argument_errors_before_any_cuda_call(entry):
    lib = N.lib()
    out = C.create_string_buffer(64)
    tail = (None, 0) if entry == "b2v_submit_tensor" else (None, C.addressof(out))

    def call(t, handle=C.c_void_p(1)):
        rc = getattr(lib, entry)(handle, None if t is None else C.byref(t), *tail)
        return rc, lib.b2v_last_error()

    for t, why in [(None, b"null"), (_tensor(dtype=4), b"unknown dtype"), (_tensor(dtype=-1), b"unknown dtype"),
                   (_tensor(fmt=4), b"unknown pixel format"), (_tensor(fmt=99), b"unknown pixel format"),
                   (_tensor(sc=0), b"stride_c"), (_tensor(sy=-64), b"stride_y"), (_tensor(sx=0), b"stride_x"),
                   (_tensor(sx=3), b"stride_x"), (_tensor(sy=65), b"stride_y"), (_tensor(dtype=N.B2V_DT_F32, sc=4098), b"stride_c"),
                   (_tensor(sy=1 << 31), b"too large"), (_tensor(sx=1 << 31), b"too large"), (_tensor(sc=1 << 48), b"too large"),
                   (_tensor(data=None), b"null"), (_tensor(data=0x1001), b"not aligned"), (_tensor(dtype=N.B2V_DT_F32, sc=4096, sx=4, data=0x1002), b"not aligned")]:
        rc, msg = call(t)
        assert rc == N.B2V_EINVAL and why in msg, (why, rc, msg)
    rc, msg = call(_tensor(), handle=None)
    assert rc == N.B2V_EINVAL and b"null" in msg


def test_uint8_strides_need_no_alignment():
    """With one-byte elements every positive stride and every address passes the argument checks: the call gets as far as the
    null handle."""
    rc = N.lib().b2v_submit_tensor(None, C.byref(_tensor(dtype=N.B2V_DT_U8, sx=3, sy=65, sc=1, data=0x1001)), None, 0)
    assert rc == N.B2V_EINVAL and b"null handle" in N.lib().b2v_last_error()


def test_struct_layout_matches_the_header():
    src = open(os.path.join(ROOT, "include", "b2video.h")).read()
    body = re.search(r"typedef struct b2v_tensor \{(.*?)\} b2v_tensor;", src, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    ctype = {"const void*": C.c_void_p, "int32_t": C.c_int32, "int64_t": C.c_int64}
    fields = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        m = re.match(r"(const void\*|int32_t|int64_t)\s+(.*)", decl)
        fields += [(name.strip(), ctype[m.group(1)]) for name in m.group(2).split(",")]
    assert fields == list(N.B2VTensor._fields_)
    assert C.sizeof(N.B2VTensor) == 40 and N.B2VTensor.stride_c.offset == 16
    enum = re.search(r"enum \{ (B2V_DT_U8 = 0, B2V_DT_F16 = 1, B2V_DT_BF16 = 2, B2V_DT_F32 = 3) \};", src)
    assert enum and (N.B2V_DT_U8, N.B2V_DT_F16, N.B2V_DT_BF16, N.B2V_DT_F32) == (0, 1, 2, 3)
    assert {k: v for k, v in DTYPES.items()} == {"u8": (0, 1), "f16": (1, 2), "bf16": (2, 2), "f32": (3, 4)}


def _fields(t):
    return t.data, t.dtype, t.pixel_format, t.stride_c, t.stride_y, t.stride_x


def test_pointer_strides_and_dtype():
    # contiguous (C, H, W) fp16, strides not given
    t, st = tensor_frame_args(Cai((3, 100, 200), "<f2", ptr=BASE), 200, 100, 0)
    assert _fields(t) == (BASE, N.B2V_DT_F16, N.B2V_PIX_RGB, 40000, 400, 2) and st == 0
    # (H, W, C) fp32, four channels, blue first
    t, _ = tensor_frame_args(Cai((100, 200, 4), "<f4", ptr=BASE), 200, 100, 0, channels="BGRA", layout="HWC")
    assert _fields(t) == (BASE, N.B2V_DT_F32, N.B2V_PIX_BGRA, 4, 3200, 16)
    # a window of a padded planar uint8 surface
    t, _ = tensor_frame_args(Cai((3, 120, 260), "|u1", strides=(40960, 320, 1), ptr=BASE), 200, 100, 0, channels="BGR", origin=(7, 11))
    assert _fields(t) == (BASE + 11 * 320 + 7, N.B2V_DT_U8, N.B2V_PIX_BGR, 40960, 320, 1)
    # picture 2 of an (N, 3, H, W) fp16 batch: the caller's slice is a (3, H, W) view further into the allocation
    plane = 100 * 200 * 2
    t, _ = tensor_frame_args(Cai((3, 100, 200), "<f2", strides=(plane, 400, 2), ptr=BASE + 2 * 3 * plane), 200, 100, 0)
    assert _fields(t) == (BASE + 6 * plane, N.B2V_DT_F16, N.B2V_PIX_RGB, plane, 400, 2)
    # the same picture of a channels_last batch: still layout="CHW", the strides say the rest
    t, _ = tensor_frame_args(Cai((3, 100, 200), "<f2", strides=(2, 1200, 6), ptr=BASE), 198, 100, 0, origin=(2, 0))
    assert _fields(t) == (BASE + 12, N.B2V_DT_F16, N.B2V_PIX_RGB, 2, 1200, 6)
    # stream rules are device_frame_args'
    assert tensor_frame_args(Cai((3, 10, 20), "<f4", stream=0x1234), 20, 10, 0)[1] == 0x1234
    assert tensor_frame_args(Cai((3, 10, 20), "<f4", stream=0x1234), 20, 10, 0, stream=0x99)[1] == 0x99


def test_bfloat16_has_no_typestr():
    """torch exports bfloat16 as '<V2'.  It is bf16 when the object is a torch tensor of that dtype, or when the caller says so."""
    with pytest.raises(TypeError):
        tensor_frame_args(Cai((3, 10, 20), "<V2"), 20, 10, 0)
    t, _ = tensor_frame_args(Cai((3, 10, 20), "<V2"), 20, 10, 0, dtype="bf16")
    assert (t.dtype, t.stride_x) == (N.B2V_DT_BF16, 2)
    with pytest.raises(TypeError):
        tensor_frame_args(Cai((3, 10, 20), "<f2"), 20, 10, 0, dtype="bf16")       # the array says fp16
    with pytest.raises(TypeError):
        tensor_frame_args(Cai((3, 10, 20), "<V4"), 20, 10, 0, dtype="bf16")


def test_bfloat16_of_a_torch_tensor(monkeypatch):
    """A stand-in for torch in sys.modules: the product looks the module up there and never imports it."""
    class Tensor(Cai):
        def __init__(self, dtype, *a, **kw):
            super().__init__(*a, **kw)
            self.dtype, self.device = dtype, types.SimpleNamespace(type="cuda", index=0)
    fake = types.SimpleNamespace(Tensor=Tensor, bfloat16="bf16-dtype", float16="f16-dtype",
                                 cuda=types.SimpleNamespace(current_stream=lambda dev: types.SimpleNamespace(cuda_stream=0x77)))
    monkeypatch.setitem(sys.modules, "torch", fake)
    t, st = tensor_frame_args(Tensor(fake.bfloat16, (3, 10, 20), "<V2"), 20, 10, 0)
    assert (t.dtype, st) == (N.B2V_DT_BF16, 0x77)
    with pytest.raises(TypeError):
        tensor_frame_args(Tensor(fake.float16, (3, 10, 20), "<V2"), 20, 10, 0)     # a 2-byte void that is not bfloat16
    with pytest.raises(TypeError):
        tensor_frame_args(Cai((3, 10, 20), "<V2"), 20, 10, 0)                      # not a torch tensor at all


@pytest.mark.parametrize("frame,kw,exc", [
    (Cai((3, 10, 20), "<f8"), {}, TypeError),                                       # fp64
    (Cai((3, 10, 20), "<u2"), {}, TypeError),                                       # ints other than uint8
    (Cai((3, 10, 20), "|i1"), {}, TypeError),
    (Cai((3, 10, 20), ">f4"), {}, TypeError),                                       # big-endian
    (Cai((1, 10, 20), "<f2"), {}, ValueError),                                      # one and two channels
    (Cai((2, 10, 20), "<f2"), {}, ValueError),
    (Cai((4, 10, 20), "<f2"), {}, ValueError),                                      # four channels called RGB
    (Cai((3, 10, 20), "<f2"), {"channels": "RGBA"}, ValueError),
    (Cai((10, 20, 3), "<f2"), {}, ValueError),                                      # (H, W, C) called CHW
    (Cai((2, 3, 10, 20), "<f2"), {}, ValueError),                                   # a batch
    (Cai((10, 20), "<f2"), {}, ValueError),
    (Cai((3, 10, 20), "<f2", strides=(400, -40, 2)), {}, ValueError),               # flipped rows
    (Cai((3, 10, 20), "<f2", strides=(0, 40, 2)), {}, ValueError),                  # a channel broadcast
    (Cai((3, 10, 20), "<f2", strides=(400, 1 << 31, 2)), {}, ValueError),
    (Cai((3, 10, 20), "<f2"), {"origin": (1, 0)}, ValueError),                      # window outside the array
    (Cai((3, 10, 20), "<f2"), {"origin": (0, 1)}, ValueError),
    (Cai((3, 10, 20), "<f2"), {"origin": (-1, 0)}, ValueError),
    (Cai((3, 10, 20), "<f2"), {"channels": "YUV"}, ValueError),
    (Cai((3, 10, 20), "<f2"), {"layout": "WHC"}, ValueError),
    (Cai((3, 10, 20), "<f2"), {"dtype": "f64"}, ValueError),
    (Cai((3, 10, 20), "<f2"), {"dtype": "f32"}, TypeError),                         # the caller's dtype disagrees with the array
    (np.zeros((3, 10, 20), np.float32), {}, TypeError),                             # host array
])
def test_rejected_before_the_c_call(frame, kw, exc):
    with pytest.raises(exc):
        tensor_frame_args(frame, 20, 10, 0, **kw)


class _Fake(_FakeSession):
    def submit_tensor(self, frame, **kw):
        self.calls.append(("tensor", frame, kw))


def test_screen_capture_routes_tensor_sources_to_submit_tensor():
    class Src(TensorFrameSource):
        channels, layout, dtype, stream = "BGR", "HWC", "bf16", 0x55

        def frame(self, index):
            return None if index >= 1 else "tensor0"

    class Packed(DeviceFrameSource):
        def frame(self, index):
            return "surface0"
    cs = ScreenCapture(Src())
    cs._origin = (37, 150)
    fake = _Fake()
    assert cs._encode_next(fake, 0) and not cs._encode_next(fake, 1)
    (kind, frame, kw), = fake.calls
    assert (kind, frame) == ("tensor", "tensor0")
    assert {k: kw[k] for k in ("channels", "layout", "dtype", "stream", "origin")} == \
        {"channels": "BGR", "layout": "HWC", "dtype": "bf16", "stream": 0x55, "origin": (37, 150)}
    fake = _Fake()
    assert ScreenCapture(Packed())._encode_next(fake, 0)
    assert fake.calls[0][0] == "device" and set(fake.calls[0][2]) == {"pixel_format", "stream", "origin", "capture_ns"}
