"""Thin object wrapper over one libb2video session handle (include/b2video.h).

One Session = one encoder instance on one GPU: what one `pixelflux.ScreenCapture`
is in the reference (one per display, selkies.py:3178-3181).  Used by
pixelflux_compat.ScreenCapture, bench.py and the tests.
"""
from __future__ import annotations

import ctypes as C
import sys
import threading
from typing import Callable, Optional

import numpy as np

from . import _native as N


class EncodedFrame:
    __slots__ = ("data", "frame_id", "is_key", "qp", "pts90k", "capture_ns", "y_start", "height")

    def __init__(self, data: bytes, frame_id: int, is_key: bool, qp: int, pts90k: int, capture_ns: int, y_start: int = 0, height: int = 0):
        self.data = data
        self.frame_id = frame_id
        self.is_key = is_key
        self.qp = qp
        self.pts90k = pts90k
        self.capture_ns = capture_ns
        self.y_start, self.height = y_start, height


# pixel formats of device frames: name -> (B2V_PIX_* code, bytes per pixel); the name is the byte order in memory
PIXEL_FORMATS = {"BGRA": (N.B2V_PIX_BGRA, 4), "RGBA": (N.B2V_PIX_RGBA, 4), "BGR": (N.B2V_PIX_BGR, 3), "RGB": (N.B2V_PIX_RGB, 3)}


def _array_interface(frame, device: int, entry: str):
    """The `__cuda_array_interface__` of `frame`, and torch when `frame` is one of its tensors (else None).  The checks every
    device entry shares: there is such an interface, a torch tensor is on the session's device, no mask."""
    cai = getattr(frame, "__cuda_array_interface__", None)
    if cai is None:
        raise TypeError(f"{type(frame).__name__} has no __cuda_array_interface__: {entry} takes device arrays (host frames go "
                        "through submit())")
    torch = sys.modules.get("torch")                   # a torch tensor means torch is imported already; never import it here
    if torch is not None and not isinstance(frame, torch.Tensor):
        torch = None
    if torch is not None and (frame.device.type != "cuda" or frame.device.index != device):
        raise ValueError(f"frame is on {frame.device}, the session runs on cuda:{device}")
    if cai.get("mask") is not None:
        raise ValueError("masked arrays are not supported")
    return cai, torch


def _producer_stream(frame, cai, torch, stream) -> int:
    """The producer's stream handle, by the rules in device_frame_args."""
    if stream is not None:
        return int(getattr(stream, "cuda_stream", stream))
    if "stream" in cai:
        return 0 if cai["stream"] is None else int(cai["stream"])
    if torch is not None:
        return torch.cuda.current_stream(frame.device).cuda_stream
    return 0


def _window(origin, width: int, height: int, full_w: int, full_h: int):
    x, y = (int(v) for v in origin)
    if x < 0 or y < 0 or x + width > full_w or y + height > full_h:
        raise ValueError(f"window {width}x{height} at ({x}, {y}) lies outside the {full_w}x{full_h} frame")
    return x, y


def device_frame_args(frame, width: int, height: int, device: int, pixel_format: str = "BGRA", origin=(0, 0), stream=None):
    """Reads the `__cuda_array_interface__` of `frame` and returns the arguments of b2v_submit_device for its `width` x `height`
    window at `origin` = (x, y): (pointer, pitch in bytes, B2V_PIX_* code, producer stream handle).  The array must be uint8,
    (H, W, 4) or (H, W, 3) as the format says, with packed pixels and any row stride.  Raises TypeError / ValueError for
    anything else; the library checks the memory itself (device, allocation bounds).

    Producer stream: `stream` when given (a handle, or an object with `.cuda_stream` such as torch.cuda.Stream); else the
    array's own `stream` entry (version 3 of the interface: None = nothing to wait for, 1 = the legacy default stream, 2 = the
    per-thread default stream, otherwise a handle); else, for a torch tensor, torch's current stream on its device; else the
    legacy default stream."""
    if pixel_format not in PIXEL_FORMATS:
        raise ValueError(f"unknown pixel format {pixel_format!r} (one of {', '.join(PIXEL_FORMATS)})")
    fmt, bpp = PIXEL_FORMATS[pixel_format]
    cai, torch = _array_interface(frame, device, "submit_device")
    if str(cai["typestr"])[1:] != "u1":
        raise TypeError(f"frame dtype {cai['typestr']!r}: uint8 pixels are needed")
    shape = tuple(int(v) for v in cai["shape"])
    if len(shape) != 3 or shape[2] != bpp:
        raise ValueError(f"frame shape {shape}: {pixel_format} needs (H, W, {bpp})")
    strides = cai.get("strides")
    pitch, px, ch = (shape[1] * bpp, bpp, 1) if strides is None else (int(v) for v in strides)
    if px != bpp or ch != 1:
        raise ValueError(f"frame strides {tuple(strides)}: pixels must be packed ({bpp}, 1); only the row stride is free")
    if pitch < shape[1] * bpp or pitch >= 1 << 31:
        raise ValueError(f"row stride {pitch} does not hold a row of {shape[1]} pixels")
    x, y = _window(origin, width, height, shape[1], shape[0])
    ptr = int(cai["data"][0]) + y * pitch + x * bpp
    return ptr, pitch, fmt, _producer_stream(frame, cai, torch, stream)


# element types of tensors: name -> (B2V_DT_* code, bytes per element), and the typestr (without byte order) that names each
DTYPES = {"u8": (N.B2V_DT_U8, 1), "f16": (N.B2V_DT_F16, 2), "bf16": (N.B2V_DT_BF16, 2), "f32": (N.B2V_DT_F32, 4)}
_TYPESTR = {"u1": "u8", "f2": "f16", "f4": "f32"}


def tensor_frame_args(frame, width: int, height: int, device: int, *, channels: str = "RGB", layout: str = "CHW", dtype=None,
                      origin=(0, 0), stream=None):
    """Reads the `__cuda_array_interface__` of a 3-D `frame` and returns (filled b2v_tensor, producer stream handle) for its
    `width` x `height` window at `origin` = (x, y).  `channels` ("RGB", "BGR", "RGBA", "BGRA") says how many channels there are
    and whether channel 0 is red or blue; `layout` ("CHW" or "HWC") only names the axes of the shape: the strides are the
    array's own, so channels_last tensors, slices of a batch and other views need no flag.  Elements are uint8, or fp16 / bf16
    / fp32 in [0, 1] (include/b2video.h has the rounding).  bf16 has no typestr: a 2-byte void element ('<V2', what torch
    exports) is taken as bf16 when `frame` is a torch tensor of dtype bfloat16 or the caller says dtype="bf16".  `dtype`, when
    given, must agree with the array otherwise.  Producer stream: as device_frame_args."""
    if channels not in PIXEL_FORMATS:
        raise ValueError(f"unknown channel order {channels!r} (one of {', '.join(PIXEL_FORMATS)})")
    if layout not in ("CHW", "HWC"):
        raise ValueError(f"unknown layout {layout!r} (CHW or HWC)")
    if dtype is not None and dtype not in DTYPES:
        raise ValueError(f"unknown dtype {dtype!r} (one of {', '.join(DTYPES)})")
    fmt, nch = PIXEL_FORMATS[channels]
    cai, torch = _array_interface(frame, device, "submit_tensor")
    code = str(cai["typestr"])[1:]
    if code == "V2" and (dtype == "bf16" or (torch is not None and frame.dtype == torch.bfloat16)):
        name = "bf16"
    elif code in _TYPESTR and str(cai["typestr"])[0] in "<|=":
        name = _TYPESTR[code]
    else:
        raise TypeError(f"frame dtype {cai['typestr']!r}: elements are uint8, float16, bfloat16 or float32")
    if dtype is not None and dtype != name:
        raise TypeError(f"frame dtype {cai['typestr']!r} is not the {dtype} the caller names")
    dt, elem = DTYPES[name]
    shape = tuple(int(v) for v in cai["shape"])
    if len(shape) != 3:
        raise ValueError(f"frame shape {shape}: a 3-D array is needed ({layout}); encode a batch one tensor at a time")
    strides = cai.get("strides")
    strides = (shape[1] * shape[2] * elem, shape[2] * elem, elem) if strides is None else tuple(int(v) for v in strides)
    (c, sc), (h, sy), (w, sx) = (sorted(zip(layout, shape, strides))[i][1:] for i in range(3))      # "C" < "H" < "W"
    if c != nch:
        raise ValueError(f"frame shape {shape}: {channels} in {layout} needs {nch} channels, the array has {c}")
    if min(sc, sy, sx) <= 0 or max(sy, sx) >= 1 << 31:
        raise ValueError(f"frame strides {strides}: every stride must be positive (rows and columns below 2 GiB)")
    x, y = _window(origin, width, height, w, h)
    t = N.B2VTensor(int(cai["data"][0]) + y * sy + x * sx, dt, fmt, sc, sy, sx)
    return t, _producer_stream(frame, cai, torch, stream)


class Session:
    def __init__(self, width: int, height: int, *, dst_width: int = 0, dst_height: int = 0, fps: float = 60.0,
                 device: int = 0, rc_mode: int = N.B2V_RC_CBR, bitrate_kbps: int = 8000, crf: int = 26,
                 gop: int = -1, slice_rows: int = 0, paintover_trigger_frames: int = 0, paintover_crf: int = 18, paintover_burst_frames: int = 1, idr_slice_mbs: int = 0, stripe_rows: int = 0, header_mode: int = N.B2V_HDR_NONE, ring_slots: int = 4,
                 flags: int = 0, on_frame: Optional[Callable[[C.POINTER(N.B2VFrame)], None]] = None,
                 collect: bool = True):
        self._lib = N.lib()
        self.device = device
        self.width, self.height = width, height
        self.dst_width, self.dst_height = dst_width or width, dst_height or height
        self.frames: list[EncodedFrame] = []
        self._collect = collect
        self._on_frame = on_frame
        self._lock = threading.Lock()
        s = N.B2VSettings()
        s.src_w, s.src_h, s.dst_w, s.dst_h = width, height, dst_width, dst_height
        s.fps, s.device, s.rc_mode, s.bitrate_kbps, s.crf = float(fps), device, rc_mode, bitrate_kbps, crf
        s.gop, s.slice_rows, s.header_mode, s.ring_slots, s.flags = gop, slice_rows, header_mode, ring_slots, flags
        s.paintover_trigger_frames, s.paintover_crf, s.stripe_rows = paintover_trigger_frames, paintover_crf, stripe_rows
        s.paintover_burst_frames, s.idr_slice_mbs = paintover_burst_frames, idr_slice_mbs
        # keep alive for the lifetime of the handle.  With nothing to deliver to Python the library gets no callback at all: a
        # ctypes callback takes the GIL on the output thread for every picture, which costs the submitting thread its pace.
        self._cb = N.FRAME_CB(self._callback) if (on_frame is not None or collect) else N.FRAME_CB()
        h = C.c_void_p()
        N.check(self._lib.b2v_create(C.byref(s), self._cb, None, C.byref(h)))
        self._h = h

    # -- native callback (fires on the library's output thread) ------------------------------
    def _callback(self, fptr, _user):
        if self._on_frame is not None:
            self._on_frame(fptr)
        if self._collect:
            f = fptr.contents
            rec = EncodedFrame(C.string_at(f.data, f.size), f.frame_id, bool(f.is_key), f.qp, f.pts90k, f.capture_ns, f.y_start, f.height)
            with self._lock:
                self.frames.append(rec)

    # -- ingest ---------------------------------------------------------------------------------
    def submit(self, bgra: np.ndarray, capture_ns: int = 0) -> None:
        """Copy one (H,W,4) uint8 BGRA frame into the next pinned ring slot and enqueue it."""
        assert bgra.dtype == np.uint8 and bgra.shape == (self.height, self.width, 4), bgra.shape
        slot = C.c_int32(-1)
        p = self._lib.b2v_ring_acquire(self._h, C.byref(slot))
        if not p:
            N.check(N.B2V_ESTATE)
        C.memmove(p, np.ascontiguousarray(bgra).ctypes.data, self.width * self.height * 4)
        N.check(self._lib.b2v_ring_submit(self._h, slot.value, self.width * 4, capture_ns))

    def acquire(self):
        """Zero-copy ingest: returns (slot, numpy view of the pinned slot) to fill in place."""
        slot = C.c_int32(-1)
        p = self._lib.b2v_ring_acquire(self._h, C.byref(slot))
        if not p:
            N.check(N.B2V_ESTATE)
        buf = (C.c_ubyte * (self.width * self.height * 4)).from_address(p)
        return slot.value, np.frombuffer(buf, np.uint8).reshape(self.height, self.width, 4)

    def release_slot(self, slot: int) -> None:
        """Give the most recently acquired slot back without encoding it."""
        N.check(self._lib.b2v_ring_release(self._h, slot))

    def submit_slot(self, slot: int, capture_ns: int = 0) -> None:
        N.check(self._lib.b2v_ring_submit(self._h, slot, self.width * 4, capture_ns))

    def resident_upload(self, index: int, bgra: np.ndarray) -> None:
        bgra = np.ascontiguousarray(bgra)
        N.check(self._lib.b2v_resident_upload(self._h, index, bgra.ctypes.data, self.width * 4))

    def submit_resident(self, index: int, capture_ns: int = 0) -> None:
        N.check(self._lib.b2v_submit_resident(self._h, index, capture_ns))

    def submit_device(self, frame, *, pixel_format: str = "BGRA", stream=None, origin=(0, 0), capture_ns: int = 0) -> None:
        """Encode the `width` x `height` window at `origin` = (x, y) of a frame in device memory of the session's GPU, without a
        copy: `frame` is any object with `__cuda_array_interface__` (torch, CuPy, Numba), uint8 (H, W, 4) for BGRA / RGBA or
        (H, W, 3) for BGR / RGB.  The conversion runs in stream order after the producer's stream (see device_frame_args), and
        that stream waits for it in turn: the frame may be overwritten in stream order as soon as this returns."""
        ptr, pitch, fmt, handle = device_frame_args(frame, self.width, self.height, self.device, pixel_format, origin, stream)
        N.check(self._lib.b2v_submit_device(self._h, ptr, pitch, fmt, handle, capture_ns))

    def submit_tensor(self, frame, *, channels: str = "RGB", layout: str = "CHW", dtype=None, stream=None, origin=(0, 0),
                      capture_ns: int = 0) -> None:
        """Encode the `width` x `height` window at `origin` of a 3-D tensor in device memory of the session's GPU as it is: uint8,
        or fp16 / bf16 / fp32 in [0, 1], planar or interleaved, any strides (tensor_frame_args).  The colour conversion
        quantises the elements as it reads them: no clamp / scale / cast / permute pass is needed in front.  Stream order as
        submit_device."""
        t, handle = tensor_frame_args(frame, self.width, self.height, self.device, channels=channels, layout=layout, dtype=dtype,
                                      origin=origin, stream=stream)
        N.check(self._lib.b2v_submit_tensor(self._h, C.byref(t), handle, capture_ns))

    def flush(self) -> None:
        N.check(self._lib.b2v_flush(self._h))

    # -- control ----------------------------------------------------------------------------------
    def set_framerate(self, fps: float) -> None:
        N.check(self._lib.b2v_set_framerate(self._h, float(fps)))

    def set_bitrate_kbps(self, kbps: int) -> None:
        N.check(self._lib.b2v_set_bitrate_kbps(self._h, int(kbps)))

    def set_qp(self, qp: int) -> None:
        N.check(self._lib.b2v_set_qp(self._h, int(qp)))

    def set_resolution(self, width: int, height: int, dst_width: int = 0, dst_height: int = 0) -> None:
        N.check(self._lib.b2v_set_resolution(self._h, width, height, dst_width, dst_height))
        self.width, self.height = width, height
        self.dst_width, self.dst_height = dst_width or width, dst_height or height

    def set_gop(self, frames: int) -> None:
        """Key-frame distance in pictures from the next submit on (<= 0: key frames only on request)."""
        N.check(self._lib.b2v_set_gop(self._h, int(frames)))

    def request_idr(self) -> None:
        N.check(self._lib.b2v_request_idr(self._h))

    # -- introspection ----------------------------------------------------------------------------
    def coded_size(self):
        w, h = C.c_int32(), C.c_int32()
        N.check(self._lib.b2v_coded_size(self._h, C.byref(w), C.byref(h)))
        return w.value, h.value

    def stats(self) -> dict:
        st = N.B2VStats()
        N.check(self._lib.b2v_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    def reset_stats(self) -> None:
        N.check(self._lib.b2v_reset_stats(self._h))

    def csc_nv12(self, bgra: np.ndarray):
        """Synchronous fused CSC(+scale): returns (Y (dh,dw), UV (dh/2,dw)) uint8."""
        bgra = np.ascontiguousarray(bgra)
        assert bgra.shape == (self.height, self.width, 4)
        dw, dh = self.dst_width, self.dst_height
        out = np.empty(dw * dh * 3 // 2, np.uint8)
        N.check(self._lib.b2v_csc_nv12(self._h, bgra.ctypes.data, self.width * 4, out.ctypes.data))
        return out[: dw * dh].reshape(dh, dw), out[dw * dh:].reshape(dh // 2, dw)

    def csc_nv12_tensor(self, frame, **kw):
        """csc_nv12 of a device tensor read in place; keywords as submit_tensor (without capture_ns)."""
        t, handle = tensor_frame_args(frame, self.width, self.height, self.device, **kw)
        dw, dh = self.dst_width, self.dst_height
        out = np.empty(dw * dh * 3 // 2, np.uint8)
        N.check(self._lib.b2v_csc_nv12_tensor(self._h, C.byref(t), handle, out.ctypes.data))
        return out[: dw * dh].reshape(dh, dw), out[dw * dh:].reshape(dh // 2, dw)

    def recon(self):
        cw, ch = self.coded_size()
        out = np.empty(cw * ch * 3 // 2, np.uint8)
        N.check(self._lib.b2v_get_recon(self._h, out.ctypes.data))
        return out[: cw * ch].reshape(ch, cw), out[cw * ch:].reshape(ch // 2, cw)

    def bench_csc(self, n_resident: int, iters: int) -> float:
        ms = C.c_float()
        N.check(self._lib.b2v_bench_csc(self._h, n_resident, iters, C.byref(ms)))
        return float(ms.value)

    def bench_csc_burst(self, n_resident: int, iters: int) -> float:
        ms = C.c_float()
        N.check(self._lib.b2v_bench_csc_burst(self._h, n_resident, iters, C.byref(ms)))
        return float(ms.value)

    def timer_start(self) -> None:
        N.check(self._lib.b2v_timer_start(self._h))

    def timer_stop(self) -> float:
        ms = C.c_float()
        N.check(self._lib.b2v_timer_stop(self._h, C.byref(ms)))
        return float(ms.value)

    def take_frames(self) -> list:
        with self._lock:
            out, self.frames = self.frames, []
        return out

    def close(self) -> None:
        if self._h:
            self._lib.b2v_destroy(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
