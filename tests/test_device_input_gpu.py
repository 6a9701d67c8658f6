"""GPU: frames already in device memory (b2v_submit_device, Session.submit_device, pixelflux_compat.DeviceFrameSource).

Every pixel format on every CSC path must give the oracle's bitstream for the same pixels in BGRA order; the producer's stream
and the library's are ordered both ways; regions of one surface feed separate captures; bad frames are refused before anything
is enqueued, and each refusal leaves the session encoding."""
import ctypes as C
import glob
import os
import threading

import numpy as np
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.pixelflux_compat import CaptureSettings, DeviceFrameSource, ScreenCapture
from selkies_b200.session import Session
from tests import longrun_scripts as L
from tests import device_scenario as D
from tests import scenario, synth
from tests.scenario import CBR, CQP, Config, picture

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

FORMATS = ["BGRA", "RGBA", "BGR", "RGB"]
W, H = 320, 192


def frames(n=6):
    return [L.desktop(W, H, t) for t in range(n - 1)] + [L.noise(W, H, 7)]


# ---- parity through the two-sided driver ----------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("rc", [(CQP, 0), (CQP, 28), (CBR, 28)], ids=["qp0", "qp28", "cbr"])
def test_parity_every_format(fmt, rc):
    """Pitch = width * bytes per pixel: the 1:1 fast kernel of the format.  QP 0 turns a one-LSB CSC difference into a level."""
    cfg = D.DeviceConfig(W, H, rc_mode=rc[0], qp=rc[1], kbps=2000, pixel_format=fmt)
    D.run(cfg, scenario.stream(frames()))


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("margin", [(16, 4), (3, 1)], ids=["padded_pitch", "unaligned_origin"])
def test_parity_surface_window(fmt, margin):
    """(16, 4): a padded pitch with the window still 16-byte aligned (fast kernels).  (3, 1): the window starts 12 B (4-byte
    formats) or 9 B (3-byte formats) past a 16-byte boundary and the pitch is no multiple of 16: the general kernel."""
    cfg = D.DeviceConfig(W, H, qp=0, pixel_format=fmt, margin=margin)
    D.run(cfg, scenario.stream(frames()))


@pytest.mark.parametrize("fmt", FORMATS)
def test_resize_through_every_csc_path(fmt):
    """1:1, ragged, scaled with 10 KB and 80 KB tiles, the general scaled kernel and an upscale (tests/longrun_scripts.py)."""
    cfg = D.DeviceConfig(L.W, L.H, rc_mode=CQP, qp=28, pixel_format=fmt)
    D.run(cfg, L.resize_script())


@pytest.mark.parametrize("fmt", ["BGRA", "RGB"])
def test_striped(fmt):
    cfg = D.DeviceConfig(**{**vars(L.STRIPED), "pixel_format": fmt})
    L.check_striped(scenario.pictures(D.run(cfg, L.striped())))


@pytest.mark.parametrize("fmt", ["RGBA", "BGR"])
def test_live_cbr(fmt):
    cfg = D.DeviceConfig(**{**vars(L.LIVE_CBR), "pixel_format": fmt})
    L.check_live_cbr(scenario.pictures(D.run(cfg, L.live_cbr())))


class _Alternating(D.DeviceGpuSide):
    """Even pictures through the host ring, odd ones from device memory, in one session."""

    n = 0

    def picture(self, frame):
        self.n += 1
        if self.n % 2:
            self.s.submit(frame)
        else:
            super().picture(frame)


def test_ring_and_device_submits_alternate():
    cfg = D.DeviceConfig(W, H, rc_mode=CBR, kbps=1500, pixel_format="RGB", margin=(3, 2))
    with D.gpu_side(_Alternating):
        scenario.run(cfg, scenario.stream([L.desktop(W, H, t) for t in range(12)]))


# ---- ScreenCapture with a DeviceFrameSource ---------------------------------------------------------------------------------
class _Surfaces(DeviceFrameSource):
    """Pre-built surfaces, one per picture, then the end of the stream; `done` is set when the capture asks past the end."""

    def __init__(self, surfaces, pixel_format):
        self.surfaces, self.pixel_format, self.done = surfaces, pixel_format, threading.Event()

    def frame(self, index):
        if index >= len(self.surfaces):
            self.done.set()
            return None
        return self.surfaces[index]


def _capture(settings, source):
    got = []

    def cb(ptr, _u):
        r = ptr.contents
        got.append(bytes(r.data[:r.size]))
    cap = ScreenCapture(source)
    cap.start_capture(settings, cb)
    return cap, got


def _settings(w, h, x=0, y=0, **kw):
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.capture_x, cs.capture_y, cs.target_fps = w, h, x, y, 240.0
    cs.h264_crf = 28
    for k, v in kw.items():
        setattr(cs, k, v)
    return cs


@pytest.mark.parametrize("fmt", ["BGRA", "RGB"])
def test_regions_of_one_surface(fmt):
    """Two captures read different windows of the same device surfaces; the x offset 37 is not a multiple of 4 pixels."""
    SW, SH, n = 704, 416, 5
    full = [synth.desktop(SW, SH, t) for t in range(n)]
    surfaces = [D.device_surface(f, fmt) for f in full]
    regions = [(0, 0, 320, 192), (37, 150, 352, 224)]
    caps = []
    for x, y, w, h in regions:
        src = _Surfaces(surfaces, fmt)
        caps.append((src,) + _capture(_settings(w, h, x, y), src))
    for src, cap, _ in caps:
        assert src.done.wait(30)
        cap.stop_capture()
    for (x, y, w, h), (_, _, got) in zip(regions, caps):
        crop = [np.ascontiguousarray(f[y:y + h, x:x + w]) for f in full]
        want = scenario.pictures(scenario.run(Config(w, h, qp=28), scenario.stream(crop), gpu=False))
        assert len(got) == n
        for g, x_ in zip(got, want):
            assert g[10:] == x_.au, f"region at ({x}, {y}), picture {x_.index}"


def test_jpeg_from_a_device_source():
    """output_mode 0: every delivered stripe is the oracle's JFIF file of that picture's stripe."""
    fmt, SW, SH, x0, y0, w, h, n, q = "RGB", 400, 240, 6, 20, 320, 192, 3, 70
    full = [synth.desktop(SW, SH, t) for t in range(n)]
    src = _Surfaces([D.device_surface(f, fmt) for f in full], fmt)
    cap, got = _capture(_settings(w, h, x0, y0, output_mode=0, jpeg_quality=q), src)
    assert src.done.wait(30)
    cap.stop_capture()
    rows = ((h // 16 + 7) // 8) * 16
    assert sum(int.from_bytes(g[0:2], "big") == 0 for g in got) == -(-h // rows)     # picture 0 sends every stripe
    for g in got:
        k, ys = int.from_bytes(g[0:2], "big"), int.from_bytes(g[2:4], "big")
        crop = np.ascontiguousarray(full[k][y0 + ys: y0 + min(h, ys + rows), x0: x0 + w])
        assert g[4:] == oracle.jpeg_encode_bgra(crop, q), (k, ys)


# ---- stream order -------------------------------------------------------------------------------------------------------------
SLEEP_CYCLES = 400_000_000          # about 0.2 s at H100 clocks: the host is long back before the producer's stream gets going


@pytest.mark.parametrize("in_flight", [0, 3])
@pytest.mark.parametrize("fmt", ["BGRA", "BGR"])
def test_stream_order_with_the_producer(fmt, in_flight):
    """On the producer's stream: sleep, write frame A, submit, write frame B into the same tensor.  The picture is A's: the CSC
    waited for the write of A, and the write of B waited for the CSC.  The submit returns while the sleep still runs."""
    before = [L.desktop(W, H, 20 + t) for t in range(in_flight)]
    a, b = L.desktop(W, H, 40), L.noise(W, H, 41)
    want = scenario.pictures(scenario.run(Config(W, H, qp=0), scenario.stream(before + [a]), gpu=False))
    da, db = (torch.from_numpy(D.reorder(f, fmt)).cuda() for f in (a, b))
    surf = torch.zeros_like(da)
    others = [D.device_surface(f, fmt) for f in before]
    torch.cuda.synchronize()
    prod = torch.cuda.Stream()
    with Session(W, H, rc_mode=N.B2V_RC_CQP, crf=0) as s:
        for t in others:
            s.submit_device(t, pixel_format=fmt)           # in flight on the session, not flushed
        with torch.cuda.stream(prod):
            torch.cuda._sleep(SLEEP_CYCLES)
            surf.copy_(da)
            s.submit_device(surf, pixel_format=fmt)        # torch's current stream: prod
            still_sleeping = not prod.query()
            surf.copy_(db)
        s.flush()
        got = s.take_frames()
    assert still_sleeping, "submit_device waited for the producer's stream"
    assert [g.data for g in got] == [x.au for x in want]
    assert torch.equal(surf, db)


def test_explicit_stream_handle_wins():
    """An explicit stream argument beats torch's current stream."""
    a = L.desktop(W, H, 3)
    want = scenario.pictures(scenario.run(Config(W, H, qp=28), [picture(a)], gpu=False))
    surf = torch.zeros((H, W, 4), dtype=torch.uint8, device="cuda")
    da = torch.from_numpy(np.array(a)).cuda()
    torch.cuda.synchronize()
    prod = torch.cuda.Stream()
    with Session(W, H, rc_mode=N.B2V_RC_CQP, crf=28) as s:
        with torch.cuda.stream(prod):
            torch.cuda._sleep(SLEEP_CYCLES)
            surf.copy_(da)
        s.submit_device(surf, stream=prod)               # called on the default stream, ordered after prod
        s.flush()
        got = s.take_frames()
    assert [g.data for g in got] == [want[0].au]


# ---- rejections ---------------------------------------------------------------------------------------------------------------
def _cudart():
    """The CUDA runtime torch loaded (raw cudaMalloc / cudaHostAlloc, no caching allocator in between)."""
    torch.cuda.init()
    for name in ["libcudart.so.12"] + glob.glob(os.path.join(os.path.dirname(torch.__file__), "..", "nvidia", "cuda_runtime", "lib", "libcudart.so*")):
        try:
            rt = C.CDLL(name)
            break
        except OSError:
            continue
    else:
        pytest.skip("no CUDA runtime library to allocate raw buffers with")
    rt.cudaMalloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t]
    rt.cudaHostAlloc.argtypes = [C.POINTER(C.c_void_p), C.c_size_t, C.c_uint]
    rt.cudaFree.argtypes = rt.cudaFreeHost.argtypes = [C.c_void_p]
    rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
    return rt


def _granularity():
    """Minimum mapping granularity of device 0 (cuMemGetAllocationGranularity), or None if the driver does not say."""
    class Prop(C.Structure):       # CUmemAllocationProp: type, requestedHandleTypes, location {type, id}, win32 handle, allocFlags
        _fields_ = [("type", C.c_int), ("handle", C.c_int), ("loc_type", C.c_int), ("loc_id", C.c_int), ("win32", C.c_void_p),
                    ("compression", C.c_ubyte), ("gpu_direct", C.c_ubyte), ("usage", C.c_ushort), ("reserved", C.c_ubyte * 4)]
    try:
        cu = C.CDLL("libcuda.so.1")
    except OSError:
        return None
    p = Prop(type=1, handle=0, loc_type=1, loc_id=0)      # pinned, device 0
    g = C.c_size_t()
    return g.value if cu.cuMemGetAllocationGranularity(C.byref(g), C.byref(p), 0) == 0 else None


def _einval(s, ptr, pitch, fmt, why):
    rc = s._lib.b2v_submit_device(s._h, ptr, pitch, fmt, None, 0)
    msg = (s._lib.b2v_last_error() or b"").decode()
    assert rc == N.B2V_EINVAL, (rc, msg)
    assert why in msg, msg


def test_rejections_leave_the_session_encoding():
    rt = _cudart()
    w, h = W, H
    f0, f1 = L.desktop(w, h, 5), L.desktop(w, h, 6)
    row = w * 4
    want = scenario.pictures(scenario.run(Config(w, h, qp=28), [picture(f0), picture(f1)], gpu=False))
    good = D.device_surface(f0)
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=28) as s:
        gp = good.data_ptr()
        # arguments, before any CUDA call
        _einval(s, gp, row, 4, "unknown pixel format")
        _einval(s, gp, row - 4, N.B2V_PIX_BGRA, "pitch")
        _einval(s, gp + 2, row, N.B2V_PIX_BGRA, "multiples of 4")
        _einval(s, gp, row + 2, N.B2V_PIX_RGBA, "multiples of 4")
        # pinned host memory the device could read (a broken check would only cost a slow read of the right pixels)
        hp = C.c_void_p()
        assert rt.cudaHostAlloc(C.byref(hp), row * h, 0) == 0
        try:
            C.memmove(hp.value, np.ascontiguousarray(f0).ctypes.data, row * h)
            _einval(s, hp.value, row, N.B2V_PIX_BGRA, "not device memory")
        finally:
            rt.cudaFreeHost(hp)
        # a raw allocation one row short of the frame, sized so that the missing row still lies in the allocation's last
        # mapping granule: a broken check would read stale bytes of mapped memory, never fault
        gran = _granularity()
        assert gran == 2 << 20, gran                      # Hopper's granule; the sizes below rely on it
        size = row * (h - 1)                              # h - 1 rows; the missing last row ends inside the same granule
        assert (size + row - 1) // gran == (size - 1) // gran
        dp = C.c_void_p()
        assert rt.cudaMalloc(C.byref(dp), size) == 0
        try:
            assert rt.cudaMemcpy(dp, np.ascontiguousarray(f0).ctypes.data, size, 1) == 0
            _einval(s, dp.value, row, N.B2V_PIX_BGRA, "past the end of its allocation")
        finally:
            rt.cudaFree(dp)
        s.submit_device(good)
        s.submit_device(D.device_surface(f1, "RGB"), pixel_format="RGB")
        s.flush()
        got = s.take_frames()
    assert [g.data for g in got] == [x.au for x in want]


def test_rejects_memory_of_another_gpu():
    if torch.cuda.device_count() < 2 or not torch.cuda.can_device_access_peer(0, 1):
        pytest.skip("needs a second GPU with peer access to the first")
    f0 = L.desktop(W, H, 2)
    rt = _cudart()
    rt.cudaSetDevice(0)
    rc = rt.cudaDeviceEnablePeerAccess(1, 0)                # a broken check then reads the peer's memory, never faults
    if rc not in (0, 704):                                  # 704: cudaErrorPeerAccessAlreadyEnabled
        pytest.skip(f"cudaDeviceEnablePeerAccess(1) failed ({rc})")
    other = D.device_surface(f0, device=1)
    want = scenario.pictures(scenario.run(Config(W, H, qp=28), [picture(f0)], gpu=False))
    with Session(W, H, rc_mode=N.B2V_RC_CQP, crf=28, device=0) as s:
        with pytest.raises(ValueError):
            s.submit_device(other)                                     # torch names the device: refused in Python
        _einval(s, other.data_ptr(), W * 4, N.B2V_PIX_BGRA, "device 1")   # and by the library
        s.submit_device(D.device_surface(f0, device=0))
        s.flush()
        got = s.take_frames()
    assert [g.data for g in got] == [want[0].au]
