"""GPU: device tensors as a model leaves them (b2v_submit_tensor, Session.submit_tensor, pixelflux_compat.TensorFrameSource).

The quantisation rule is checked over every fp16 and bf16 bit pattern; every dtype, channel order and memory form on every
CSC path must give the oracle's output for the quantised pixels; the producer's stream and the library's are ordered both ways;
bad tensors are refused before anything is enqueued, and each refusal leaves the session encoding."""
import ctypes as C
import threading

import numpy as np
import pytest

import oracle
from selkies_b200 import _native as N
from selkies_b200.pixelflux_compat import CaptureSettings, ScreenCapture, TensorFrameSource
from selkies_b200.session import Session, tensor_frame_args
from tests import device_scenario as D
from tests import longrun_scripts as L
from tests import scenario, synth
from tests import tensor_scenario as T
from tests.scenario import CBR, CQP, Config, picture
from tests.test_device_input_gpu import SLEEP_CYCLES, _cudart, _granularity

torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

W, H = 320, 192


def frames(n=6):
    return [L.desktop(W, H, t) for t in range(n - 1)] + [L.noise(W, H, 7)]


# ---- the quantisation rule ------------------------------------------------------------------------------------------------
def _grey_luma(values, form):
    """JFIF luma of the grey picture whose three channels all hold `values` (H, W): the sample itself, as 4899 + 9617 + 1868 =
    2^14.  "CHW": the planar kernel; "HWC": the general kernel's per-element loader."""
    h, w = values.shape
    t = values.cuda().expand(3, h, w).contiguous() if form == "CHW" else values.cuda()[..., None].expand(h, w, 3).contiguous()
    with Session(w, h, flags=N.B2V_FLAG_JPEG) as s:
        y, _ = s.csc_nv12_tensor(t, layout=form)
    return y


@pytest.mark.parametrize("form", ["CHW", "HWC"])
@pytest.mark.parametrize("dtype", ["f16", "bf16"])
def test_every_16_bit_pattern(dtype, form):
    """All 65 536 patterns: NaNs, infinities, negatives, subnormals and every tie."""
    v = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(T.torch_dtype(dtype)).reshape(256, 256)
    want = T.quantise(v.float().numpy())
    assert len(np.unique(want)) == 256
    assert np.array_equal(_grey_luma(v, form), want)


@pytest.mark.parametrize("form", ["CHW", "HWC"])
def test_fp32_specials_ties_and_random_patterns(form):
    rng = np.random.default_rng(3)
    bits = rng.integers(0, 1 << 32, 1024 * 1024, dtype=np.uint64).astype(np.uint32)
    ties = ((np.arange(255, dtype=np.float64) + 0.5) / 255).astype(np.float32).view(np.uint32)
    near = (ties[:, None].astype(np.int64) + np.arange(-4, 5)[None, :]).astype(np.uint32).ravel()          # +-4 ulp of every tie
    special = np.array([0.0, -0.0, 1.0, -1.0, 2.0, np.inf, -np.inf, np.nan, -np.nan, 1e-45, -1e-45, 1e-38, 0.5, 1 / 255, 254.5 / 255,
                        np.nextafter(np.float32(1), np.float32(0)), np.nextafter(np.float32(1), np.float32(2)), 3.4e38], np.float32).view(np.uint32)
    bits[:near.size] = near
    bits[near.size:near.size + special.size] = special
    x = bits.view(np.float32).reshape(1024, 1024)
    assert np.array_equal(_grey_luma(torch.from_numpy(x.copy()), form), T.quantise(x))


# ---- colour conversion parity through the hook --------------------------------------------------------------------------------
def _csc_case(dtype, channels, form, w, h, margin=(0, 0), dst=(0, 0), jpeg=False, seed=1):
    t, q = T.host_tensor(synth.noise(w, h, seed), dtype, channels, noise_seed=seed)
    dev, layout = T.device_tensor(t, form, margin)
    with Session(w, h, dst_width=dst[0], dst_height=dst[1], flags=N.B2V_FLAG_JPEG if jpeg else N.B2V_FLAG_NO_ENCODE) as s:
        y, uv = s.csc_nv12_tensor(dev, channels=channels, layout=layout, origin=margin)
    oy, ouv = oracle.csc_nv12(q, dst_w=dst[0], dst_h=dst[1], matrix=1 if jpeg else 0)
    assert np.array_equal(y, oy), "luma"
    assert np.array_equal(uv, ouv), "chroma"


@pytest.mark.parametrize("channels", ["RGB", "BGR", "RGBA", "BGRA"])
@pytest.mark.parametrize("dtype", T.DTYPES)
def test_csc_planar_and_interleaved(dtype, channels):
    """Contiguous (C, H, W) at a width that is a multiple of every kernel's unit, from a 16-byte aligned allocation: the planar
    kernel.  (H, W, C): uint8 is a packed frame and takes its kernels, floats take the general one."""
    _csc_case(dtype, channels, "CHW", 320, 64)
    _csc_case(dtype, channels, "HWC", 320, 64)


@pytest.mark.parametrize("dtype", T.DTYPES)
def test_csc_windows_and_views(dtype):
    _csc_case(dtype, "RGB", "CHW", 320, 64, margin=(16, 3))         # padded pitch and plane stride, window still 16-byte aligned
    _csc_case(dtype, "BGR", "CHW", 320, 64, margin=(3, 1))          # window off 16-byte alignment: general kernel
    _csc_case(dtype, "RGB", "CHW", 324, 64)                         # width no multiple of 8 or 16 pixels
    _csc_case(dtype, "RGB", "CHW", 130, 34)                         # ragged
    _csc_case(dtype, "BGR", "NHWC", 320, 64)                        # channels_last view of a batch
    _csc_case(dtype, "RGBA", "HWC", 322, 64, margin=(5, 2))
    _csc_case(dtype, "RGB", "CHW", 320, 64, jpeg=True)              # JFIF matrix
    _csc_case(dtype, "BGR", "HWC", 128, 64, jpeg=True)


@pytest.mark.parametrize("dtype", T.DTYPES)
@pytest.mark.parametrize("sw,sh,dw,dh", [(640, 360, 320, 180), (160, 96, 320, 192), (1920, 1080, 320, 180)], ids=["down", "up", "tile80k"])
def test_csc_scaled(dtype, sw, sh, dw, dh):
    """Quantise first, then the integer bilinear blend: the tiled kernel (10 KB and 80 KB of shared memory) and an upscale."""
    _csc_case(dtype, "RGB", "CHW", sw, sh, dst=(dw, dh))
    if sw <= 640:
        _csc_case(dtype, "BGR", "HWC", sw, sh, dst=(dw, dh), margin=(2, 1))


def test_csc_scaled_by_the_general_kernel():
    """A 4K source down by 12: the tile's footprint no longer fits shared memory."""
    _csc_case("f16", "RGB", "CHW", 3840, 2160, dst=(320, 180))


# ---- encode parity through the two-sided driver -------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", T.DTYPES)
@pytest.mark.parametrize("rc", [(CQP, 0), (CQP, 28), (CBR, 28)], ids=["qp0", "qp28", "cbr"])
def test_parity_every_dtype(dtype, rc):
    cfg = T.TensorConfig(W, H, rc_mode=rc[0], qp=rc[1], kbps=2000, dtype=dtype)
    T.run(cfg, scenario.stream(frames()))


def test_resize_through_every_csc_path():
    cfg = T.TensorConfig(L.W, L.H, rc_mode=CQP, qp=28, dtype="f16")
    T.run(cfg, L.resize_script())


def test_striped():
    cfg = T.TensorConfig(**{**vars(L.STRIPED), "dtype": "bf16", "channels": "BGR", "noise": False})
    L.check_striped(scenario.pictures(T.run(cfg, L.striped())))


def test_live_cbr():
    cfg = T.TensorConfig(**{**vars(L.LIVE_CBR), "dtype": "f32", "form": "HWC", "noise": False})
    L.check_live_cbr(scenario.pictures(T.run(cfg, L.live_cbr())))


class _Alternating(T.TensorGpuSide):
    """Pictures through the host ring, b2v_submit_device and b2v_submit_tensor in turn, in one session."""

    n = 0

    def picture(self, frame):
        self.n += 1
        if self.n % 3 == 1:
            self.s.submit(frame)
        elif self.n % 3 == 2:
            self.s.submit_device(D.device_surface(frame, "RGB"), pixel_format="RGB")
        else:
            super().picture(frame)


def test_ring_device_and_tensor_submits_alternate():
    cfg = T.TensorConfig(W, H, rc_mode=CBR, kbps=1500, dtype="f16", margin=(8, 2))
    T.run(cfg, scenario.stream([L.desktop(W, H, t) for t in range(12)]), cls=_Alternating)


# ---- ScreenCapture with a TensorFrameSource -----------------------------------------------------------------------------------
class _Tensors(TensorFrameSource):
    def __init__(self, tensors, channels, layout):
        self.tensors, self.channels, self.layout, self.done = tensors, channels, layout, threading.Event()

    def frame(self, index):
        if index >= len(self.tensors):
            self.done.set()
            return None
        return self.tensors[index]


def _capture(src, w, h, x, y, **kw):
    cs = CaptureSettings()
    cs.capture_width, cs.capture_height, cs.capture_x, cs.capture_y, cs.target_fps, cs.h264_crf = w, h, x, y, 240.0, 28
    for k, v in kw.items():
        setattr(cs, k, v)
    got = []
    cap = ScreenCapture(src)
    cap.start_capture(cs, lambda ptr, _u: got.append(bytes(ptr.contents.data[:ptr.contents.size])))
    assert src.done.wait(30)
    cap.stop_capture()
    return got


def test_screen_capture_from_a_tensor_source():
    """A window, 37 pixels in, of bf16 (C, H, W) surfaces."""
    SW, SH, x, y, w, h, n = 448, 256, 37, 30, 320, 192, 4
    pairs = [T.host_tensor(synth.desktop(SW, SH, t), "bf16", "RGB", noise_seed=t) for t in range(n)]
    got = _capture(_Tensors([T.device_tensor(t)[0] for t, _ in pairs], "RGB", "CHW"), w, h, x, y)
    crop = [np.ascontiguousarray(q[y:y + h, x:x + w]) for _, q in pairs]
    want = scenario.pictures(scenario.run(Config(w, h, qp=28), scenario.stream(crop), gpu=False))
    assert [g[10:] for g in got] == [x_.au for x_ in want]


def test_jpeg_from_a_tensor_source():
    SW, SH, x0, y0, w, h, n, q = 400, 240, 8, 20, 320, 192, 3, 70
    pairs = [T.host_tensor(synth.desktop(SW, SH, t), "f16", "BGR", noise_seed=t) for t in range(n)]
    got = _capture(_Tensors([T.device_tensor(t, "HWC")[0] for t, _ in pairs], "BGR", "HWC"), w, h, x0, y0, output_mode=0, jpeg_quality=q)
    rows = ((h // 16 + 7) // 8) * 16
    assert sum(int.from_bytes(g[0:2], "big") == 0 for g in got) == -(-h // rows)     # picture 0 sends every stripe
    for g in got:
        k, ys = int.from_bytes(g[0:2], "big"), int.from_bytes(g[2:4], "big")
        crop = np.ascontiguousarray(pairs[k][1][y0 + ys: y0 + min(h, ys + rows), x0: x0 + w])
        assert g[4:] == oracle.jpeg_encode_bgra(crop, q), (k, ys)


# ---- stream order -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("in_flight", [0, 3])
def test_stream_order_with_the_producer(in_flight):
    """On the producer's stream: sleep, write tensor A, submit, write B into the same tensor.  The picture is A's, and the
    submit returns while the sleep still runs."""
    before = [T.host_tensor(L.desktop(W, H, 20 + t), "f16") for t in range(in_flight)]
    (ta, qa), (tb, _) = T.host_tensor(L.desktop(W, H, 40), "f16", noise_seed=1), T.host_tensor(L.noise(W, H, 41), "f16", noise_seed=2)
    want = scenario.pictures(scenario.run(Config(W, H, qp=0), scenario.stream([q for _, q in before] + [qa]), gpu=False))
    da, db = T.device_tensor(ta)[0], T.device_tensor(tb)[0]
    surf = torch.zeros_like(da)
    others = [T.device_tensor(t)[0] for t, _ in before]
    torch.cuda.synchronize()
    prod = torch.cuda.Stream()
    with Session(W, H, rc_mode=N.B2V_RC_CQP, crf=0) as s:
        for t in others:
            s.submit_tensor(t)                             # in flight on the session, not flushed
        with torch.cuda.stream(prod):
            torch.cuda._sleep(SLEEP_CYCLES)
            surf.copy_(da)
            s.submit_tensor(surf)                          # torch's current stream: prod
            still_sleeping = not prod.query()
            surf.copy_(db)
        s.flush()
        got = s.take_frames()
    assert still_sleeping, "submit_tensor waited for the producer's stream"
    assert [g.data for g in got] == [x.au for x in want]
    assert torch.equal(surf, db)


# ---- rejections ---------------------------------------------------------------------------------------------------------------
def _einval(s, t, why):
    rc = s._lib.b2v_submit_tensor(s._h, C.byref(t), None, 0)
    msg = (s._lib.b2v_last_error() or b"").decode()
    assert rc == N.B2V_EINVAL, (rc, msg)
    assert why in msg, msg


def test_rejections_leave_the_session_encoding():
    rt = _cudart()
    w, h = W, H
    (t0, q0), (t1, q1) = (T.host_tensor(L.desktop(w, h, 5 + k), "f16", noise_seed=k) for k in range(2))
    want = scenario.pictures(scenario.run(Config(w, h, qp=28), [picture(q0), picture(q1)], gpu=False))
    good = T.device_tensor(t0)[0]
    plane, row = w * h * 2, w * 2
    raw = np.ascontiguousarray(t0.permute(2, 0, 1).contiguous().view(torch.int16).numpy())
    with Session(w, h, rc_mode=N.B2V_RC_CQP, crf=28) as s:
        desc, _ = tensor_frame_args(good, w, h, 0)
        assert (desc.stride_c, desc.stride_y, desc.stride_x) == (plane, row, 2)
        # pinned host memory the device could read (a broken check would only cost a slow read of the right elements)
        hp = C.c_void_p()
        assert rt.cudaHostAlloc(C.byref(hp), 3 * plane, 0) == 0
        try:
            C.memmove(hp.value, raw.ctypes.data, 3 * plane)
            _einval(s, N.B2VTensor(hp.value, N.B2V_DT_F16, N.B2V_PIX_RGB, plane, row, 2), "not device memory")
        finally:
            rt.cudaFreeHost(hp)
        # a raw allocation whose last plane is one row short, sized so that the missing row still lies in the allocation's
        # last mapping granule: a broken check (one that forgot stride_c, say) would read mapped memory, never fault
        gran = _granularity()
        assert gran == 2 << 20, gran
        size = 3 * plane - row
        assert (size + row - 1) // gran == (size - 1) // gran
        dp = C.c_void_p()
        assert rt.cudaMalloc(C.byref(dp), size) == 0
        try:
            assert rt.cudaMemcpy(dp, raw.ctypes.data, size, 1) == 0
            _einval(s, N.B2VTensor(dp.value, N.B2V_DT_F16, N.B2V_PIX_RGB, plane, row, 2), "past the end of its allocation")
            # with its planes a row closer together the tensor ends inside the allocation: what fits is not refused
            fits = N.B2VTensor(dp.value, N.B2V_DT_F16, N.B2V_PIX_RGB, plane - row, row, 2)
            assert s._lib.b2v_csc_nv12_tensor(s._h, C.byref(fits), None, np.empty(w * h * 3 // 2, np.uint8).ctypes.data) == 0
        finally:
            rt.cudaFree(dp)
        s.submit_tensor(good)
        s.submit_tensor(T.device_tensor(t1, "HWC")[0], layout="HWC")
        s.flush()
        got = s.take_frames()
    assert [g.data for g in got] == [x.au for x in want]


def test_rejects_a_tensor_of_another_gpu():
    if torch.cuda.device_count() < 2 or not torch.cuda.can_device_access_peer(0, 1):
        pytest.skip("needs a second GPU with peer access to the first")
    rt = _cudart()
    rt.cudaSetDevice(0)
    rc = rt.cudaDeviceEnablePeerAccess(1, 0)                # a broken check then reads the peer's memory, never faults
    if rc not in (0, 704):                                  # 704: cudaErrorPeerAccessAlreadyEnabled
        pytest.skip(f"cudaDeviceEnablePeerAccess(1) failed ({rc})")
    t0, q0 = T.host_tensor(L.desktop(W, H, 2), "f16")
    other = T.device_tensor(t0, device=1)[0]
    want = scenario.pictures(scenario.run(Config(W, H, qp=28), [picture(q0)], gpu=False))
    with Session(W, H, rc_mode=N.B2V_RC_CQP, crf=28, device=0) as s:
        with pytest.raises(ValueError):
            s.submit_tensor(other)                                     # torch names the device: refused in Python
        _einval(s, N.B2VTensor(other.data_ptr(), N.B2V_DT_F16, N.B2V_PIX_RGB, W * H * 2, W * 2, 2), "device 1")
        s.submit_tensor(T.device_tensor(t0, device=0)[0])
        s.flush()
        got = s.take_frames()
    assert [g.data for g in got] == [want[0].au]
